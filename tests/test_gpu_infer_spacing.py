"""Insert-size inference (`snap paired -ins`) on the device: snapgpu_align_paired_ins against the compiled reference aligner driven
pair by pair as PairedAligner.cpp:889-925 drives it, and the drop-in `snap-aligner-gpu paired -ins` against stock `snap-aligner`."""
from __future__ import annotations

import math
import os
import subprocess

import numpy as np
import pytest

from conftest import differing_pairs

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GPU_BIN = os.path.join(ROOT, "integration", "_build", "snap-aligner-gpu")
INVALID = 0xFFFFFFFF
WIN = 1000
LAUNCHES_PER_UPDATE = 5          # include/snapgpu.h: snapgpu_align_paired_ins makes at most 5 sub-launches per update, plus 5

pytestmark = pytest.mark.gpu

# (snapgpu / reference params, paired params, filterFlags): default, `-fs -F a`, `-F a -F b`
OPTION_SETS = {
    "default": (dict(maxDist=14), dict(), 0),
    "fs_Fa": (dict(maxDist=14), dict(forceSpacing=1), 0x16),
    "Fa_Fb": (dict(maxDist=14), dict(), 0x16 | 0x8),
}


@pytest.fixture(scope="module")
def engine():
    from snap_b200 import engine as e
    if e.lib().snapgpu_device_count() < 1:
        pytest.fail("no CUDA device")
    return e


@pytest.fixture(scope="module")
def genome(tmp_path_factory, reflib):
    from snap_b200 import synth
    d = tmp_path_factory.mktemp("ins")
    contigs = synth.make_contigs(3, 200_000, seed=91, repeat_frac=0.1)
    synth.write_fasta(str(d / "ref.fa"), contigs)
    reflib.build_reference_index(reflib.SNAP_ALIGNER, str(d / "ref.fa"), str(d / "idx"))
    return contigs, str(d / "idx")


def _two_population_pairs(contigs, n, seed, same_strand_frac=0.0):
    """~85 % N(300, 30) and 15 % N(800, 60) inserts, in random order; `same_strand_frac` of the pairs get their second end
    reverse-complemented, so both ends align on one strand and add no sample."""
    from snap_b200 import synth
    n2 = int(0.15 * n)
    a = synth.make_pairs(contigs, n - n2, 100, seed=seed, insert_mean=300, insert_sd=30, chimeric_frac=0.02, n_run_frac=0.01, short_frac=0.01)
    b = synth.make_pairs(contigs, n2, 100, seed=seed + 1, insert_mean=800, insert_sd=60)
    rng = np.random.default_rng(seed)
    order = rng.permutation(n)
    flip = rng.random(n) < same_strand_frac
    reads = []
    for k, j in enumerate(order):
        src, i = (a, j) if j < n - n2 else (b, j - (n - n2))
        r0, r1 = src.read(2 * i), src.read(2 * i + 1)
        if flip[k]:
            arr = np.frombuffer(r1[0], dtype=np.uint8)
            r1 = (synth.revcomp(arr).tobytes(), r1[1][::-1])
        reads += [r0, r1]
    return synth.ReadBatch.from_lists(reads)


def _py_range(s):
    """computeSpacingDist (PairedAligner.cpp:424-458) over a sorted window of any size, in Python doubles."""
    w = len(s)
    s = [int(x) for x in s]
    s25, s75 = s[int(0.25 * w)], s[int(0.75 * w)]

    def to_int(v):           # int64 -> int, and x86-64's double -> int
        if isinstance(v, int):
            v &= 0xFFFFFFFF
            return v - (1 << 32) if v >= 1 << 31 else v
        return int(v) if -2147483649.0 < v < 2147483648.0 else -2 ** 31
    mn, mx = to_int(max(s25 - 2 * (s75 - s25), 1)), to_int(s75 + 2 * (s75 - s25))
    tot, cnt = 0.0, 0
    for x in s:
        if mn <= x <= mx:
            tot += float(x); cnt += 1
    avg = tot / cnt if cnt else math.nan
    tot = 0.0
    for x in s:
        if mn <= x <= mx:
            tot += (x - avg) * (x - avg)
    sd = math.sqrt(tot / cnt) if cnt else math.nan
    mn, mx = to_int(s25 - 3 * (s75 - s25)), to_int(s75 + 3 * (s75 - s25))
    lo, hi = avg - 4 * sd, avg + 4 * sd
    mn = to_int(lo if lo < mn else float(mn))
    mx = to_int(hi if hi > mx else float(mx))
    return max(mn, 1), mx


def _sample(r, useful, flags, force):
    """The sample pair record `r` adds (PairedAligner.cpp:822-925), or -1."""
    if not useful[0] and not useful[1]:
        return -1
    st, loc = [int(r["status"][0]), int(r["status"][1])], [int(r["location"][0]), int(r["location"][1])]
    if force and (st[0] == 1) != (st[1] == 1):
        st, loc = [0, 0], [INVALID, INVALID]

    def pf(status, too_short):
        if flags == 0:
            return True
        if too_short:
            return bool(flags & 0x10)
        return bool(flags & {0: 0x1, 1: 0x2, 2: 0x4}[status])
    p0, p1 = pf(st[0], not useful[0]), pf(st[1], not useful[1])
    if not ((p0 and p1) if flags & 0x8 else (p0 or p1)) or r["direction"][0] == r["direction"][1]:
        return -1
    return abs(loc[0] - loc[1])


def _oracle(reflib, idx, pb, kw, pkw, flags, window):
    """The reference aligner driven pair by pair with the range stock's loop would give it.  Each segment between updates is
    aligned by a fresh reference aligner holding that segment's range (a pair's result depends only on the pair and the range).
    Returns (results, [(first pair of segment, min, max)], samples)."""
    n = pb.n // 2
    useful = [(pb.lens[i] >= 50 and pb.read(i)[0].count(b"N") <= kw["maxDist"]) for i in range(pb.n)]
    ridx = reflib.RefIndex(idx)
    out = np.zeros(n, dtype=reflib.PAIRED_RESULT_DTYPE)
    mn, mx = pkw.get("minSpacing", 0), pkw.get("maxSpacing", 1000)
    segs, win, samples, p = [(0, mn, mx)], [], 0, 0
    while p < n:
        ral = reflib.RefPairedAligner(ridx, reflib.default_params_paired(**kw), reflib.default_paired_params(**{**pkw, "minSpacing": mn, "maxSpacing": mx}))
        res, _ = ral.align(pb.slice(2 * p, 2 * n))
        ral.close()
        j = p
        while j < n:
            out[j] = res[j - p]
            s = _sample(res[j - p], (useful[2 * j], useful[2 * j + 1]), flags, pkw.get("forceSpacing", 0))
            j += 1
            if s >= 0:
                win.append(s); samples += 1
                if len(win) == window:
                    mn, mx = _py_range(sorted(win))
                    mx &= 0xFFFFFFFF
                    win = []
                    segs.append((j, mn, mx))
                    break
        p = j
    return out, segs, samples


def _add(a, b):
    """Sum of two counters_dict results (the MAPQ histogram is a list)."""
    if a is None:
        return b
    return {f: (np.add(a[f], b[f]).tolist() if isinstance(a[f], list) else a[f] + b[f]) for f in a}


def _counters_by_segments(engine, gidx, pb, kw, pkw, segs):
    """What the counters must be: the plain paired entry over each segment under that segment's range."""
    n = pb.n // 2
    tot = None
    for k, (first, mn, mx) in enumerate(segs):
        last = segs[k + 1][0] if k + 1 < len(segs) else n
        if last <= first:
            continue
        al = engine.PairedAligner(gidx, engine.default_params(**{"numSeedsFromCommandLine": 8, **kw}),
                                  engine.default_paired_params(**{**pkw, "minSpacing": mn, "maxSpacing": mx}), 8192)
        _, c = al.align(pb.slice(2 * first, 2 * last))
        al.close()
        tot = _add(tot, c)
    return tot


def _ctr_equal(a, b):
    # nHashEntriesProbed is the one counter that may differ between two runs of the same launch (see DESIGN §6)
    return {k: v for k, v in a.items() if k != "nHashEntriesProbed"} == {k: v for k, v in b.items() if k != "nHashEntriesProbed"}


@pytest.fixture(scope="module")
def gidx(engine, genome):
    ix = engine.Index.open(genome[1])
    yield ix
    ix.close()


@pytest.mark.parametrize("opt", list(OPTION_SETS))
def test_ins_matches_reference_driven_pair_by_pair(engine, gidx, genome, reflib, opt):
    import torch
    kw, pkw, flags = OPTION_SETS[opt]
    pb = _two_population_pairs(genome[0], 6000, seed=17)
    n = pb.n // 2
    want, segs, samples = _oracle(reflib, genome[1], pb, kw, pkw, flags, WIN)
    assert len(segs) >= 4
    # after the first update the range excludes the long-insert population (end-to-end distance ~700): those pairs leave the
    # intersecting aligner for the single-end fallback
    assert all(1 <= mn and mx < 600 for _, mn, mx in segs[1:]), segs
    want_ctr = _counters_by_segments(engine, gidx, pb, kw, pkw, segs)
    params, pparams = engine.default_params(**{"numSeedsFromCommandLine": 8, **kw}), engine.default_paired_params(**pkw)
    al = engine.PairedAligner(gidx, params, pparams, 8192)

    def check(got, ctr, est, how):
        bad = differing_pairs(want, got)
        assert not bad, (opt, how, len(bad), bad[:5])
        st = est.get()
        assert (st["updates"], st["minSpacing"], st["maxSpacing"], st["samples"]) == (len(segs) - 1, segs[-1][1], segs[-1][2], samples), (how, st)
        assert _ctr_equal(ctr, want_ctr), (how, {k: (ctr[k], want_ctr[k]) for k in ctr if ctr[k] != want_ctr[k]})

    # one call
    est = engine.SpacingEstimator(al, flags, WIN)
    got, ctr = est.align(pb)
    check(got, ctr, est, "one call")
    est.close()
    # calls of 777 pairs
    est = engine.SpacingEstimator(al, flags, WIN)
    got = np.zeros(n, dtype=engine.PAIRED_RESULT_DTYPE)
    ctr = None
    for p in range(0, n, 777):
        r, c = est.align(pb.slice(2 * p, 2 * min(n, p + 777)))
        got[p:p + len(r)] = r
        ctr = _add(ctr, c)
    check(got, ctr, est, "calls of 777")
    est.close()
    # device-resident buffers
    est = engine.SpacingEstimator(al, flags, WIN)
    dev = torch.device("cuda:0")
    d_b = torch.from_numpy(np.ascontiguousarray(pb.bases)).to(dev)
    d_q = torch.from_numpy(np.ascontiguousarray(pb.quals)).to(dev)
    d_o = torch.from_numpy(pb.offsets.astype(np.int64)).to(dev)
    d_l = torch.from_numpy(pb.lens.astype(np.int32)).to(dev)
    d_r = torch.zeros(n * engine.PAIRED_RESULT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    d_c = torch.zeros(engine.N_COUNTERS, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    est.align_device(n, d_b.data_ptr(), d_q.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), d_r.data_ptr(), d_c.data_ptr())
    al.check()
    got = np.frombuffer(d_r.cpu().numpy().tobytes(), dtype=engine.PAIRED_RESULT_DTYPE)
    check(got, engine.counters_dict(d_c.cpu().numpy()), est, "device")
    est.close()
    # the plain entry on the same handle still uses the handle's own -s range
    plain, _ = al.align(pb.slice(0, 2 * 500))
    ral = reflib.RefPairedAligner(reflib.RefIndex(genome[1]), reflib.default_params_paired(**kw), reflib.default_paired_params(**pkw))
    ref_plain, _ = ral.align(pb.slice(0, 2 * 500))
    ral.close()
    assert differing_pairs(ref_plain, plain) == []
    al.close()


def test_ins_low_sample_rate_stays_within_the_launch_bound(engine, gidx, genome, reflib):
    """95 % of the pairs have both ends on one strand: about one pair in 20 adds a sample, so a window of 1000 spans ~20 K pairs and
    the safe sub-launches alone would not reach it."""
    kw, pkw, flags = OPTION_SETS["default"]
    pb = _two_population_pairs(genome[0], 30000, seed=23, same_strand_frac=0.95)
    n = pb.n // 2
    want, segs, samples = _oracle(reflib, genome[1], pb, kw, pkw, flags, WIN)
    assert len(segs) >= 2
    al = engine.PairedAligner(gidx, engine.default_params(**{"numSeedsFromCommandLine": 8, **kw}), engine.default_paired_params(**pkw), 32768)
    l0 = al.launch_count()
    al.align(pb.slice(0, 2 * 100))
    per_sub = al.launch_count() - l0              # kernel launches of one sub-launch (launch form of this handle)
    est = engine.SpacingEstimator(al, flags, WIN)
    l0 = al.launch_count()
    got, _ = est.align(pb)
    launches = al.launch_count() - l0
    st, tm = est.get(), est.timing()
    assert differing_pairs(want, got) == []
    assert st["updates"] == len(segs) - 1 and st["samples"] == samples
    assert tm["subLaunches"] <= LAUNCHES_PER_UPDATE * (st["updates"] + 1), tm
    assert launches <= per_sub * LAUNCHES_PER_UPDATE * (st["updates"] + 1), (launches, per_sub, st)
    est.close(); al.close()


# ---- the drop-in at stock's window (262144) ----

def _records(path):
    return sorted(l for l in open(path, "rb").read().split(b"\n") if l and not l.startswith(b"@"))


def _headers(path):
    return [l for l in open(path, "rb").read().split(b"\n") if l.startswith(b"@") and not l.startswith(b"@PG")]


def _run(binary, argv, env=None):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([binary] + argv, capture_output=True, text=True, env=e, timeout=1500)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def _stats_line(stdout, n=5):
    import re
    lines = [l for l in stdout.split("\n") if l.strip()]
    k = max(i for i, l in enumerate(lines) if "Reads/s" in l)
    toks = re.sub(r"\([^)]*\)", " ", lines[k + 1]).split()
    return [t for t in toks if t.replace(",", "").isdigit()][:n]


@pytest.fixture(scope="module")
def big_fastq(tmp_path_factory, reflib):
    """600 K pairs (two window updates at ~95 % sample rate) from the two insert populations, on a 6 Mbp genome."""
    import torch
    from snap_b200 import synth, synth_device
    d = tmp_path_factory.mktemp("insbig")
    dev = torch.device("cuda:0")
    bases, starts = synth_device.make_genome(3, 2_000_000, seed=5, device=dev)
    contigs = [bases[int(s):int(s) + 2_000_000].cpu().numpy() for s in starts]
    synth.write_fasta(str(d / "ref.fa"), contigs)
    reflib.build_reference_index(reflib.SNAP_ALIGNER, str(d / "ref.fa"), str(d / "idx"))
    n = 600_000
    n2 = int(0.15 * n)
    parts = [synth_device.make_pairs(bases, starts, 2_000_000, n - n2, 100, seed=6, insert_mean=300, insert_sd=30),
             synth_device.make_pairs(bases, starts, 2_000_000, n2, 100, seed=7, insert_mean=800, insert_sd=60)]
    b = torch.cat([p[0].view(-1, 2, 100) for p in parts]).cpu().numpy()
    q = torch.cat([p[1].view(-1, 2, 100) for p in parts]).cpu().numpy()
    order = np.random.default_rng(8).permutation(n)
    b, q = b[order], q[order]
    f1, f2 = str(d / "r1.fq"), str(d / "r2.fq")
    for w, f in ((0, f1), (1, f2)):
        with open(f, "wb") as fh:
            fh.write(b"".join(b"@p%d/%d\n%s\n+\n%s\n" % (i, w + 1, b[i, w].tobytes(), q[i, w].tobytes()) for i in range(n)))
    return str(d / "idx"), f1, f2, n, d


def test_drop_in_ins_writes_the_stock_records(big_fastq, reflib):
    if not os.path.exists(GPU_BIN):
        pytest.fail("integration/_build/snap-aligner-gpu is missing on the GPU box")
    idx, f1, f2, n, d = big_fastq
    for extra in ([], ["-F", "a", "-F", "b", "-fs"]):
        stock = str(d / "stock.sam")
        so = _run(reflib.SNAP_ALIGNER, ["paired", idx, f1, f2, "-ins", "-o", stock, "-t", "1"] + extra)
        want = _records(stock)
        for env in ({}, {"SNAPGPU_EXT_BATCH_READS": "1000"}):
            gpu = str(d / "gpu.sam")
            go = _run(GPU_BIN, ["paired", idx, f1, f2, "-ins", "-o", gpu, "-t", "1"] + extra, env=env)
            got = _records(gpu)
            assert len(got) == len(want)
            bad = [i for i in range(len(want)) if want[i] != got[i]]
            assert not bad, (extra, env, len(bad), want[bad[0]], got[bad[0]])
            assert _headers(stock) == _headers(gpu)
            assert _stats_line(so) == _stats_line(go), (extra, env)
        if not extra:
            plain = str(d / "plain.sam")
            _run(GPU_BIN, ["paired", idx, f1, f2, "-o", plain, "-t", "1"])
            other = _records(plain)
            assert len(other) == len(want)
            assert sum(1 for x, y in zip(want, other) if x != y) >= len(want) // 100


def test_drop_in_ins_with_three_threads_writes_every_pair_once(big_fastq):
    """With -t 3 each thread infers from the pairs it reads, as stock does; the result is not compared with stock's (which depends
    on the partition too), only its completeness."""
    idx, f1, f2, n, d = big_fastq
    out = str(d / "t3.sam")
    _run(GPU_BIN, ["paired", idx, f1, f2, "-ins", "-o", out, "-t", "3"])
    recs = _records(out)
    assert len(recs) == 2 * n
    names = sorted(r.split(b"\t", 1)[0] for r in recs)
    assert names == sorted(b"p%d" % i for i in range(n) for _ in range(2))
