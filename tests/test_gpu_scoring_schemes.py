"""The affine-gap forms on the device under non-default and extreme scoring schemes (`-gm -gs -go -ge -g5 -g3`), against the compiled
reference: the leaf matrix of test_scoring_schemes.py through the leaf-test kernel, then whole reads, pairs and SAM records."""
import os

import numpy as np
import pytest

import jobs as J
import warpsim_lib as ws
from conftest import differing, differing_pairs
from scheme_jobs import CARRY, SCHEMES, scheme_jobs

pytestmark = pytest.mark.gpu

WARP_FORMS = ["0", "1", "2", "5", "13"]


@pytest.fixture(scope="module")
def engine():
    from snap_b200 import engine as e
    assert e.lib().snapgpu_device_count() >= 1, "no CUDA device: the CUDA path has no fallback"
    return e


@pytest.fixture(scope="module")
def gidx(engine, small_cfg):
    ix = engine.Index.open(small_cfg.idx)
    yield ix
    ix.close()


@pytest.mark.parametrize("name", list(SCHEMES))
def test_warp_leaves_under_scheme(engine, reflib, monkeypatch, name):
    """Every warp form where sg_ag_small_scores lets the kernels take it (only the general form outside it), on 1 and 64 warps."""
    import hostsim_lib as hs
    scheme, inside = SCHEMES[name]
    assert ws.small_scores(scheme) == inside
    t, p, q, jb = scheme_jobs(240, 170 + list(SCHEMES).index(name), scheme, CARRY.get(name, 0))
    want = reflib.ag_batch(t, p, q, jb.astype(reflib.AG_JOB_DTYPE), np.array(scheme, dtype=np.int32))
    _, stale = hs.ag_batch(t, p, q, jb, J.AG_OUT, scheme)
    hist = stale != 0
    for form in (WARP_FORMS if inside else ["0"]):
        monkeypatch.setenv("SNAPGPU_TEST_AG_PACKED", form)
        for warps in (1, 64):
            got = engine.test_ag(t, p, q, jb, J.AG_OUT, scheme, warps=warps)
            bad = np.nonzero(~J.same_out(want, got) & ~hist)[0]
            assert bad.size == 0, (name, form, warps, bad.size, jb[bad[0]], want[bad[0]], got[bad[0]])
            for f in ("agScore", "textOffset", "patternOffset"):
                assert (want[f] == got[f]).all(), (name, form, warps, f)
    if name == "saturating":
        assert (want["agScore"] == 32767).sum() >= 10


def _scheme_params(matchReward, subPenalty, gapOpenPenalty, gapExtendPenalty, fivePrimeEndBonus, threePrimeEndBonus):
    return dict(matchReward=matchReward, subPenalty=subPenalty, gapOpenPenalty=gapOpenPenalty, gapExtendPenalty=gapExtendPenalty,
                fivePrimeEndBonus=fivePrimeEndBonus, threePrimeEndBonus=threePrimeEndBonus)


# (scheme, SNAPGPU_MAX_READ_LEN or None).  The aligner's guard is taken at its own maximum read length: -gm 20 passes it at the
# default 400 and fails it at 1000, where the general form runs all of pass 2 / stages 2-3.
WHOLE_READ_SCHEMES = {
    "gs200_go199": ("gs200_go199", None),      # (the aligners refuse sub > open + extend, BaseAligner.cpp:141)
    "gm128": ("gm128", None),
    "gm20": ("gm20", None),
    "gm20_general": ("gm20", "1000"),
    "gap_2_5_8_2": ("gap_2_5_8_2", None),
    "bonus_20_3": ("bonus_20_3", None),
}
_CTR_KEYS = ("totalReads", "singleHits", "multiHits", "notFound", "nHashTableLookups", "lvCalls", "affineGapCalls", "mapqHistogram")


@pytest.mark.parametrize("opt", list(WHOLE_READ_SCHEMES))
def test_whole_reads_under_scheme_match_reference(engine, gidx, small_cfg, reflib, monkeypatch, opt):
    """Both single-end launch forms (two-pass, one launch): every field and the counters."""
    name, max_len = WHOLE_READ_SCHEMES[opt]
    kw = dict(maxDist=14, **_scheme_params(*SCHEMES[name][0]))
    if max_len:
        monkeypatch.setenv("SNAPGPU_MAX_READ_LEN", max_len)
    for rname in ("noisy150", "indel100"):
        rb = small_cfg.reads[rname]
        want, wctr = reflib.RefSingleAligner(reflib.RefIndex(small_cfg.idx), reflib.default_params(**kw)).align(rb)
        for two_pass in ("1", "0"):
            monkeypatch.setenv("SNAPGPU_TWO_PASS", two_pass)
            al = engine.SingleAligner(gidx, engine.default_params(**kw), 4096)
            got, ctr = al.align(rb)
            al.close()
            assert differing(want, got) == [], (opt, rname, two_pass)
            for k in _CTR_KEYS:
                assert wctr[k] == ctr[k], (opt, rname, two_pass, k)
        assert wctr["affineGapCalls"] > 50


# Not -gs 200 -go 199 for pairs: with substitutions as dear as gaps, the traceback of a few pairs' rescoring (3 to 5 of 600 here) steps onto
# cells the call did not write, so the reference's answer is what earlier pairs of its thread left there (DESIGN.md 3, "Reference behaviour
# that is not a function of the inputs"); the device runs pairs on other warps in another order and its answer changes with the warp count.
# The host build, which runs them in the reference's order, matches it (test_scoring_schemes.py).
@pytest.mark.parametrize("opt", [o for o in WHOLE_READ_SCHEMES if o != "gs200_go199"])
def test_pairs_under_scheme_match_reference(engine, gidx, small_cfg, reflib, monkeypatch, opt):
    """Staged and one-launch paired forms."""
    name, max_len = WHOLE_READ_SCHEMES[opt]
    kw = dict(maxDist=27, **_scheme_params(*SCHEMES[name][0]))
    if max_len:
        monkeypatch.setenv("SNAPGPU_MAX_READ_LEN", max_len)
    rp, pp = reflib.default_params_paired(**kw), reflib.default_paired_params()
    for pname in ("noisy150", "clipped150"):
        pb = small_cfg.pairs[pname]
        want, _ = reflib.RefPairedAligner(reflib.RefIndex(small_cfg.idx), rp, pp).align(pb)
        for staged in ("1", "0"):
            monkeypatch.setenv("SNAPGPU_PAIRED_STAGED", staged)
            al = engine.PairedAligner(gidx, engine.default_params(**{"numSeedsFromCommandLine": 8, **kw}), engine.default_paired_params(), 2048)
            got, _ = al.align(pb)
            al.close()
            assert differing_pairs(want, got) == [], (opt, pname, staged)


def test_sam_records_under_scheme_equal_reference_binary(engine, gidx, small_cfg, reflib, tmp_path):
    """`snap single -gm 3 -gs 20 -go 30 -ge 2 -g5 20 -g3 3`: the device's SAM records (its CIGAR DP takes the options' scores) against the
    reference binary's .sam, byte for byte."""
    import subprocess
    scheme = [3, 20, 30, 2, 20, 3]
    rb = small_cfg.reads["noisy150"]
    fq = str(tmp_path / "r.fq"); out = str(tmp_path / "o.sam")
    rb.write_fastq(fq)
    flags = ["-gm", "-gs", "-go", "-ge", "-g5", "-g3"]
    argv = ["single", small_cfg.idx, fq, "-o", out, "-t", "1", "-d", "14"] + [x for f, v in zip(flags, scheme) for x in (f, str(v))]
    r = subprocess.run([reflib.SNAP_ALIGNER] + argv, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-400:] + r.stderr[-400:]
    want = [l for l in open(out, "rb").read().split(b"\n") if l and not l.startswith(b"@")]
    p = engine.default_params(maxDist=14, **_scheme_params(*scheme))
    al = engine.SingleAligner(gidx, p, 4096)
    res, _ = al.align(rb)
    al.close()
    fmt = engine.SamFormatter(gidx, p, 4096)
    got = [l for l in fmt.format(rb, [b"r%d" % i for i in range(rb.n)], res).split(b"\n") if l]
    fmt.close()
    assert len(want) == len(got) == rb.n
    bad = [i for i in range(rb.n) if want[i] != got[i]]
    assert bad == [], (len(bad), want[bad[0]], got[bad[0]])
    cigars = [l.split(b"\t")[5] for l in got]
    assert sum(1 for c in cigars if b"I" in c or b"D" in c) > 300 and sum(1 for c in cigars if b"S" in c) > 300
