"""ALT-aware `snap paired` on the device: the index of tests/alt_pairing_data.py (ALT contigs with and without a liftover file) through
the C ABI against the compiled reference, in both launch forms, both index layouts, with tiny pools (retry pass) and in any order; and
the drop-in binary with default options against stock `snap-aligner paired`."""
import os

import numpy as np
import pytest

import alt_pairing_data as AD
from conftest import differing_pairs as _differing_pairs

pytestmark = pytest.mark.gpu


def differing_pairs(want, got):
    """conftest.differing_pairs, and refSpan is not compared for pairs that were not lifted over.  A phase-4 candidate record keeps the refSpan
    its buffer slot last held (IntersectingPairedEndAligner.cpp:1134-1163 does not write it); an end that phase 4 does not rescore reports that
    value, which depends on what the aligner did before -- another pair on another warp here.  Only the liftover reads it (as the aligned span),
    and the liftover's own results are compared in full."""
    w, g = want.copy(), got.copy()
    for a in (w, g):
        a["refSpan"][(w["liftover"] == 0).all(axis=1)] = 0
    return _differing_pairs(w, g)


@pytest.fixture(scope="module")
def engine():
    from snap_b200 import engine as e
    assert e.lib().snapgpu_device_count() >= 1, "no CUDA device: the CUDA path has no fallback"
    return e


@pytest.fixture(scope="module")
def alt_data(tmp_path_factory, reflib):
    d = str(tmp_path_factory.mktemp("gpualtpair"))
    lift, nolift, cs = AD.build(d, reflib.SNAP_ALIGNER)
    return d, lift, nolift, AD.pairs(cs, 3000, seed=4244)


_SETS = {"stock": (dict(maxDist=27), dict()), "hc": (dict(maxDist=27, fivePrimeEndBonus=5, threePrimeEndBonus=5), dict(useSoftClipping=0, minAGScoreImprovement=15))}


@pytest.mark.parametrize("opt", list(_SETS))
@pytest.mark.parametrize("layout", ["bucket", "snap"])
def test_alt_aware_pairs_on_the_device_match_reference(engine, reflib, alt_data, monkeypatch, opt, layout):
    _, lift, nolift, pairs = alt_data
    kw, pkw = _SETS[opt]
    if layout == "snap":
        monkeypatch.setenv("SNAPGPU_INDEX_LAYOUT", "snap")
    for idx in (lift, nolift):
        want, _ = reflib.RefPairedAligner(reflib.RefIndex(idx), reflib.default_params_paired(**kw), reflib.default_paired_params(**pkw)).align(pairs)
        gidx = engine.Index.open(idx)
        ctrs = {}
        for staged in ("0", "1"):
            for caps in (None, ("16", "4")):
                monkeypatch.setenv("SNAPGPU_PAIRED_STAGED", staged)
                if caps:
                    monkeypatch.setenv("SNAPGPU_PAIRED_POOL_CAP", caps[0]); monkeypatch.setenv("SNAPGPU_PAIRED_CAND_CAP", caps[1])
                else:
                    monkeypatch.delenv("SNAPGPU_PAIRED_POOL_CAP", raising=False); monkeypatch.delenv("SNAPGPU_PAIRED_CAND_CAP", raising=False)
                al = engine.PairedAligner(gidx, engine.default_params(**{"numSeedsFromCommandLine": 8, **kw}), engine.default_paired_params(**pkw), 4096)
                got, ctr = al.align(pairs)
                al.close()
                bad = differing_pairs(want, got)
                assert bad == [], (opt, layout, idx, staged, caps, len(bad), bad[:5])
                if not caps:
                    ctrs[staged] = ctr
        for k in ("totalReads", "singleHits", "multiHits", "notFound", "nHashTableLookups", "lvCalls", "affineGapCalls", "mapqHistogram"):
            assert ctrs["0"][k] == ctrs["1"][k], (opt, layout, idx, k)
        if idx == lift and opt == "stock":
            assert (want["liftover"] == 1).all(axis=1).any()
        gidx.close()


def test_alt_aware_pairs_do_not_depend_on_order_or_batch_split(engine, reflib, alt_data):
    _, lift, _, pairs = alt_data
    n = pairs.n // 2
    perm = np.random.default_rng(9).permutation(n)
    order = np.stack([2 * perm, 2 * perm + 1], axis=1).ravel()
    from snap_b200 import synth
    shuffled = synth.ReadBatch.from_lists([pairs.read(int(i)) for i in order])
    gidx = engine.Index.open(lift)
    p, pp = engine.default_params(numSeedsFromCommandLine=8, maxDist=27), engine.default_paired_params()
    al = engine.PairedAligner(gidx, p, pp, 4096)
    whole, _ = al.align(pairs)
    sh, _ = al.align(shuffled)
    al.close()
    small = engine.PairedAligner(gidx, p, pp, 100)
    parts = np.concatenate([small.align(pairs.slice(2 * lo, 2 * min(n, lo + 100)))[0] for lo in range(0, n, 100)])
    small.close()
    assert differing_pairs(whole[perm], sh) == []
    assert differing_pairs(whole, parts) == []
    gidx.close()


def test_drop_in_paired_with_default_options_on_an_alt_index(tmp_path, reflib, alt_data):
    """`snap-aligner-gpu paired <index with ALT contigs> r1.fq r2.fq` with default options (ALT-aware) writes stock `snap-aligner paired`'s records
    and totals."""
    from test_integration import GPU_BIN, _records, _run, _stats_line
    if not os.path.exists(GPU_BIN):
        pytest.fail("integration/_build/snap-aligner-gpu is missing on the GPU box")
    _, lift, _, pairs = alt_data
    f1, f2 = str(tmp_path / "r1.fq"), str(tmp_path / "r2.fq")
    with open(f1, "wb") as a, open(f2, "wb") as b:
        for i in range(pairs.n // 2):
            for w, f in ((0, a), (1, b)):
                bs, q = pairs.read(2 * i + w)
                f.write(b"@p%d/%d\n%s\n+\n%s\n" % (i, w + 1, bs, q))
    stock, gpu = str(tmp_path / "stock.sam"), str(tmp_path / "gpu.sam")
    so = _run(reflib.SNAP_ALIGNER, ["paired", lift, f1, f2, "-o", stock, "-t", "1"])
    go = _run(GPU_BIN, ["paired", lift, f1, f2, "-o", gpu, "-t", "1"])
    x, y = _records(stock), _records(gpu)
    assert len(x) == pairs.n and len(y) == pairs.n
    bad = [i for i in range(len(x)) if x[i] != y[i]]
    assert not bad, (len(bad), x[bad[0]], y[bad[0]])
    assert _stats_line(so) == _stats_line(go)
