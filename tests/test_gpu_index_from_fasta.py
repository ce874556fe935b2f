"""`snap-aligner-gpu index-gpu`: a FASTA indexed on the device against stock `snap-aligner index` with the same options -- the Genome
file byte for byte, the GenomeIndex fields, the per-table used counts, every position's hits, and the SAM records stock and drop-in
`single` / `paired` write on the directory -- plus snapgpu_index_build_genome's ALT-aware pairing and the command's refusals."""
import os
import subprocess

import numpy as np
import pytest

import alt_pairing_data as AD
import buildsim_lib as hs
from test_index_relay_geometry import table_used
from test_gpu_alt_pairing import differing_pairs

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GPU_BIN = os.path.join(ROOT, "integration", "_build", "snap-aligner-gpu")


def _run(argv, env=None, ok=True):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(argv, capture_output=True, text=True, env=e, timeout=900)
    if ok:
        assert r.returncode == 0, (argv, r.stdout[-3000:] + r.stderr[-3000:])
    return r


def _records(path):
    return sorted(l for l in open(path, "rb").read().split(b"\n") if l and not l.startswith(b"@"))


def _genome_bases(directory):
    g = open(os.path.join(directory, "Genome"), "rb").read()
    lines = g.split(b"\n", 1 + int(g.split(b"\n", 1)[0].split()[1]))
    return np.frombuffer(lines[-1], dtype=np.uint8)


@pytest.fixture(scope="module")
def data(small_cfg, reflib, tmp_path_factory):
    from snap_b200 import synth
    d = str(tmp_path_factory.mktemp("idxgpu"))
    AD.build(d, reflib.SNAP_ALIGNER)                                  # writes ref.fa and alt.sam beside the stock indexes
    cs = AD.contigs()
    out = {"small": (small_cfg.fasta, small_cfg.contigs), "alt": (os.path.join(d, "ref.fa"), cs)}
    fq = {}
    for name, (_, contigs) in out.items():
        single = os.path.join(d, name + "_r.fq")
        synth.make_reads(contigs, 600, 150, seed=71, sub_rate=0.02, ins_rate=0.002, del_rate=0.002, n_run_frac=0.05).write_fastq(single)
        pairs = AD.pairs(contigs, 600, seed=72)
        f1, f2 = os.path.join(d, name + "_1.fq"), os.path.join(d, name + "_2.fq")
        with open(f1, "wb") as a, open(f2, "wb") as b:
            for i in range(pairs.n // 2):
                for w, f in ((0, a), (1, b)):
                    bs, q = pairs.read(2 * i + w)
                    f.write(b"@p%d/%d\n%s\n+\n%s\n" % (i, w + 1, bs, q))
        fq[name] = (single, f1, f2)
    return d, out, fq, os.path.join(d, "alt.sam")


CASES = {
    "default": ("small", []),
    "s20": ("small", ["-s", "20"]),
    "s20_large": ("small", ["-s", "20", "-large"]),
    "s24_key4": ("small", ["-s", "24", "-keysize", "4"]),
    "s16_loc4": ("small", ["-s", "16", "-locationSize", "4"]),
    "s22_h06": ("small", ["-s", "22", "-h", "0.6"]),
    "p500": ("small", ["-p500"]),
    "bspace_off": ("small", ["-bSpace-"]),
    "alt_lift": ("alt", ["-s", "20", "LIFT"]),
    "alt_lift_default": ("alt", ["LIFT"]),
    "alt_nolift": ("alt", ["-s", "20"]),
    "alt_autoalt_off": ("alt", ["-s", "20", "-AutoAlt-"]),
    "alt_maxaltsize": ("alt", ["-s", "20", "-maxAltContigSize", "15000"]),
}


def _both(reflib, data, case, env=None):
    d, out, _, alt_sam = data
    which, opts = CASES[case]
    opts = [a for o in opts for a in (["-altLiftoverFile", alt_sam] if o == "LIFT" else [o])]
    fasta = out[which][0]
    want, got = os.path.join(d, case + "_stock"), os.path.join(d, case + "_gpu" + ("_env" if env else ""))
    if not os.path.exists(os.path.join(want, "GenomeIndexHash")):
        _run([reflib.SNAP_ALIGNER, "index", fasta, want, "-t8"] + opts)
    r = _run([GPU_BIN, "index-gpu", fasta, got] + opts, env=env)
    assert "device build" in r.stdout + r.stderr
    return want, got


def _same_index(reflib, want, got, contigs_bases):
    assert open(os.path.join(want, "Genome"), "rb").read() == open(os.path.join(got, "Genome"), "rb").read()
    a, b = open(os.path.join(want, "GenomeIndex")).read().split(), open(os.path.join(got, "GenomeIndex")).read().split()
    assert [a[i] for i in (0, 1, 2, 4, 5, 6, 8, 9)] == [b[i] for i in (0, 1, 2, 4, 5, 6, 8, 9)], (a, b)
    assert np.array_equal(table_used(want), table_used(got))
    seed_len = int(a[4])
    bases = contigs_bases
    seeds = np.ascontiguousarray(np.lib.stride_tricks.sliding_window_view(bases, seed_len)[:bases.size - seed_len - 1])
    hw, hg = hs.BsIndex(want), hs.BsIndex(got)
    for s in range(0, len(seeds), 50000):
        chunk = np.ascontiguousarray(seeds[s:s + 50000])
        n1, h1 = hw.lookup(chunk, len(chunk))
        n2, h2 = hg.lookup(chunk, len(chunk))
        assert np.array_equal(n1, n2), s
        k = np.minimum(n1, 512)
        mask = np.arange(512)[None, None, :] < k[:, :, None]
        assert np.array_equal(np.where(mask, h1, 0), np.where(mask, h2, 0)), s
    rw, rg = reflib.RefIndex(want), reflib.RefIndex(got)                # the unmodified reference's loader and lookupSeed32
    for i in range(0, len(seeds), 211):
        x, y = rw.lookup(seeds[i].tobytes()), rg.lookup(seeds[i].tobytes())
        assert x[:2] == y[:2] and np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3]), i


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_index_gpu_matches_stock_index(reflib, data, tmp_path, case):
    if not os.path.exists(GPU_BIN):
        pytest.fail("integration/_build/snap-aligner-gpu is missing on the GPU box")
    want, got = _both(reflib, data, case)
    _same_index(reflib, want, got, _genome_bases(want))
    single, f1, f2 = data[2][CASES[case][0]]
    recs = {}
    for tag, binary, idx in (("stock_on_stock", reflib.SNAP_ALIGNER, want), ("stock_on_gpu", reflib.SNAP_ALIGNER, got), ("gpu_on_gpu", GPU_BIN, got),
                             ("gpu_on_stock", GPU_BIN, want)):
        s, p = str(tmp_path / (tag + "_s.sam")), str(tmp_path / (tag + "_p.sam"))
        _run([binary, "single", idx, single, "-o", s, "-t", "1", "-d", "14"])
        _run([binary, "paired", idx, f1, f2, "-o", p, "-t", "1"])
        recs[tag] = (_records(s), _records(p))
    for tag in ("stock_on_gpu", "gpu_on_gpu", "gpu_on_stock"):
        assert recs[tag][0] == recs["stock_on_stock"][0], (case, tag, "single")
        assert recs[tag][1] == recs["stock_on_stock"][1], (case, tag, "paired")
    if case == "alt_lift":
        g = open(os.path.join(got, "Genome"), "rb").read(4096)
        assert b"12000M4I9000M3D8997M600S" in g


@pytest.mark.gpu
def test_index_gpu_in_forced_passes_writes_the_same_index(reflib, data):
    want, got = _both(reflib, data, "alt_lift", env={"SNAPGPU_BUILD_PASSES": "3"})
    _same_index(reflib, want, got, _genome_bases(want))


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["host", "device"])
def test_build_genome_aligns_alt_aware_like_the_stock_directory(reflib, data, monkeypatch, form):
    """snapgpu_index_build_genome with the ALT fixture's contig descriptors (parsed from the stock Genome file), not saved: ALT-aware
    pairs field for field equal to the stock directory opened on the device and to the reference, in both launch forms."""
    from snap_b200 import engine
    import torch
    d = data[0]
    lift = os.path.join(d, "idx_lift")
    g = open(os.path.join(lift, "Genome"), "rb").read()
    n = int(g.split(b"\n", 1)[0].split()[1])
    lines = g.split(b"\n")[1:1 + n]
    contigs = []
    for ln in lines:
        f = ln.split(b" ")
        name_len = int(f[5])
        rest = ln.split(b" ", 7)[7]
        name, cigar = rest[:name_len], rest[name_len + 1:]
        contigs.append(dict(name=name, beginningLocation=int(f[0]), isAlt=int(f[1], 16) & 1, originalContigNumber=int(f[2]),
                            projBeginningLocation=int(f[3]), projIsRC=int(f[4], 16) & 1, projCigar=None if cigar == b"*" else cigar))
    assert any(c["projCigar"] for c in contigs)
    bases = _genome_bases(lift)
    if form == "host":
        built = engine.Index.build_genome(bases, contigs, seed_len=20)
    else:
        t = torch.from_numpy(bases.copy()).cuda()
        built = engine.Index.build_genome(bases.size, contigs, seed_len=20, d_bases_ptr=t.data_ptr())
    opened = engine.Index.open(lift)
    pairs = AD.pairs(AD.contigs(), 3000, seed=4244)
    want, _ = reflib.RefPairedAligner(reflib.RefIndex(lift), reflib.default_params_paired(maxDist=27), reflib.default_paired_params()).align(pairs)
    assert (want["liftover"] == 1).all(axis=1).any()
    for staged in ("0", "1"):
        monkeypatch.setenv("SNAPGPU_PAIRED_STAGED", staged)
        got = {}
        for tag, ix in (("built", built), ("opened", opened)):
            al = engine.PairedAligner(ix, engine.default_params(numSeedsFromCommandLine=8, maxDist=27), engine.default_paired_params(), 4096)
            got[tag], _ = al.align(pairs)
            al.close()
        assert differing_pairs(want, got["built"]) == [], staged
        assert differing_pairs(got["opened"], got["built"]) == [], staged
    built.close(); opened.close()


@pytest.mark.gpu
def test_build_genome_refuses_bad_descriptors_and_snap_layout_geometry(data, monkeypatch, tmp_path):
    from snap_b200 import engine
    bases = np.full(50_000, ord("A"), dtype=np.uint8)
    bases[:2000] = ord("n")
    rng = np.random.default_rng(3)
    bases[2000:48000] = np.frombuffer(b"ACGT", dtype=np.uint8)[rng.integers(0, 4, 46000)]
    base = dict(projBeginningLocation=0, projIsRC=0, projCigar=None)
    for contigs, msg in (([dict(name=b"a", beginningLocation=2000, isAlt=1, originalContigNumber=0, **base),
                           dict(name=b"b", beginningLocation=25000, isAlt=0, originalContigNumber=1, **base)], "ALT contigs must come last"),
                         ([dict(name=b"a", beginningLocation=2000, isAlt=0, originalContigNumber=0, **base),
                           dict(name=b"b", beginningLocation=25000, isAlt=1, originalContigNumber=1, projBeginningLocation=2000, projIsRC=0,
                                projCigar=b"100M5Q")], "malformed projection CIGAR")):
        with pytest.raises(engine.SnapGpuError) as e:
            engine.Index.build_genome(bases, contigs, seed_len=20)
        assert msg in str(e.value)
    monkeypatch.setenv("SNAPGPU_INDEX_LAYOUT", "snap")
    ix = engine.Index.build(bases, [2000], seed_len=20)
    with pytest.raises(engine.SnapGpuError) as e:
        ix.save_ex(str(tmp_path / "x"), key_bytes=5)
    assert "SNAPGPU_INDEX_LAYOUT=snap" in str(e.value)
    ix.save(str(tmp_path / "y"))                                     # the default options still save
    ix.close()


REFUSALS = [
    (["-H/tmp/hist"], "-H"),
    (["-s", "16"], "-locationSize 4"),
    (["-s", "20", "-locationSize", "5"], "-locationSize 4"),
    (["-s", "15", "-locationSize", "4"], "16 to 24"),
    (["-s", "25"], "16 to 24"),
]


@pytest.mark.parametrize("opts,msg", REFUSALS, ids=["H", "loc5_auto", "loc5", "s15", "s25"])
def test_index_gpu_refusals(tmp_path, opts, msg):
    """Refused by name with exit status 1 before any device work (so they need no GPU)."""
    if not os.path.exists(GPU_BIN):
        pytest.skip("integration/_build/snap-aligner-gpu not built")
    fa = tmp_path / "r.fa"
    fa.write_bytes(b">c\n" + b"ACGT" * 100 + b"\n")
    r = _run([GPU_BIN, "index-gpu", str(fa), str(tmp_path / "o")] + opts, ok=False)
    assert r.returncode == 1, r.stdout + r.stderr
    assert msg in r.stdout + r.stderr
    assert not os.path.exists(tmp_path / "o" / "GenomeIndexHash")
