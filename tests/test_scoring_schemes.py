"""Every affine-gap form under non-default and extreme scoring schemes (`-gm -gs -go -ge -g5 -g3`), against the compiled reference.

The scalar form (host build) and the warp forms the kernels run (snap_b200/csrc/sg_warp_ag*.cuh, on the SIMT emulator of
tests/hostsim/warpsim.h) over jobs sized for each scheme (tests/scheme_jobs.py): large substitution penalties and match rewards,
large gap penalties, both edges of sg_ag_small_scores and cells that saturate at 32767.  Where the guard holds every form must
match the reference; where it does not, the kernels run only the general int form, and that one must match under every scheme.
Then whole reads and pairs on the host build, and the global CIGAR DP of the output stage, under the schemes with large scores."""
import functools

import numpy as np
import pytest

import hostsim_lib as hs
import jobs as J
import warpsim_lib as ws
from conftest import differing, differing_pairs
from scheme_jobs import CARRY, SCHEMES, scheme_jobs

N_JOBS = 240
WARP_FORMS = [0, 1, 2, 5, 13]      # 0 general int form; 1 packed + narrow-band rows; 2 unrolled packed; 5 duo narrow band (13: H in the arena)


@functools.lru_cache(maxsize=None)
def _case(name):
    """(jobs, reference answers, history-dependent flags, scalar form's answers) of a scheme; shared by its forms."""
    from oracle import reflib
    scheme = SCHEMES[name][0]
    t, p, q, jb = scheme_jobs(N_JOBS, 70 + list(SCHEMES).index(name), scheme, CARRY.get(name, 0))
    want = reflib.ag_batch(t, p, q, jb.astype(reflib.AG_JOB_DTYPE), np.array(scheme, dtype=np.int32))
    scalar, stale = hs.ag_batch(t, p, q, jb, J.AG_OUT, scheme)
    return (t, p, q, jb), want, stale != 0, scalar


def _assert_same(want, got, hist, jb, what):
    """Bit for bit except the history-dependent jobs (see test_ag_fuzz), which must still agree on score and offsets."""
    bad = np.nonzero(~J.same_out(want, got) & ~hist)[0]
    assert bad.size == 0, (what, "%d of %d jobs differ" % (bad.size, jb.size), jb[bad[0]], want[bad[0]], got[bad[0]])
    for f in ("agScore", "textOffset", "patternOffset"):
        bad = np.nonzero(want[f] != got[f])[0]
        assert bad.size == 0, (what, f, jb[bad[0]], want[bad[0]], got[bad[0]])


@pytest.mark.parametrize("name", list(SCHEMES))
def test_guard_side_of_each_scheme(name):
    """sg_ag_small_scores as the kernels call it: a change to the guard shows up here before it changes which form runs."""
    scheme, inside = SCHEMES[name]
    assert ws.small_scores(scheme) == inside, (name, scheme)


@pytest.mark.parametrize("name", list(SCHEMES))
def test_scalar_form_matches_reference(reflib, name):
    """The scalar form of the host build; and proof that each scheme's jobs reach what they are there for."""
    (t, p, q, jb), want, hist, scalar = _case(name)
    _assert_same(want, scalar, hist, jb, "scalar")
    assert hist.sum() <= 0.06 * jb.size
    assert ((jb["banded"] == 0) & (jb["patternLen"] <= 192)).sum() > 60
    assert ((jb["banded"] != 0) & (jb["w"] <= 15) & (jb["w"] >= 0)).sum() > 60
    assert (((jb["banded"] != 0) & (jb["w"] > 15)) | ((jb["banded"] == 0) & (jb["patternLen"] > 192))).sum() > 40
    scheme = SCHEMES[name][0]
    gm = scheme[0]
    assert (want["agScore"] > gm * 0.5 * jb["patternLen"]).sum() > 0.3 * jb.size       # many jobs align, at scores the scheme scales
    if name == "saturating":
        assert (want["agScore"] == 32767).sum() >= 10
    if name.startswith("top_in"):
        assert (want["agScore"] > 11000).sum() >= 3


@pytest.mark.parametrize("name,form", [(n, f) for n in SCHEMES for f in WARP_FORMS if f == 0 or SCHEMES[n][1]])
def test_warp_forms_match_reference(reflib, name, form):
    """Form 0 under every scheme; the specialised forms where the guard lets the kernels take them (outside it they never run)."""
    scheme = SCHEMES[name][0]
    (t, p, q, jb), want, hist, _ = _case(name)
    got = ws.ag_batch(t, p, q, jb, J.AG_OUT, scheme, form)
    _assert_same(want, got, hist, jb, "form %d" % form)


# `snap single` / `snap paired` with large scores: pass 2 / stages 2-3 around the gate gapOpen / (sub - gapExtend), and (-gm) the general
# form running all of the affine-gap rescoring on the device.  The aligners refuse sub > open + extend (BaseAligner.cpp:141), so -gs 200
# comes with -go 199.
WHOLE_READ_SCHEMES = {
    "gs200_go199": dict(subPenalty=200, gapOpenPenalty=199),
    "gm128": dict(matchReward=128),
    "gm20": dict(matchReward=20),
}


@pytest.mark.parametrize("opt", list(WHOLE_READ_SCHEMES))
def test_whole_reads_under_large_scores_match_reference(reflib, small_cfg, opt):
    p = reflib.default_params(maxDist=14, **WHOLE_READ_SCHEMES[opt])
    ridx, hidx = reflib.RefIndex(small_cfg.idx), hs.HsIndex(small_cfg.idx)
    n_ag = 0
    for name, two_pass in (("noisy150", False), ("indel100", True), ("long250", False)):
        rb = small_cfg.reads[name]
        ral = reflib.RefSingleAligner(ridx, p)
        want, wctr = ral.align(rb)
        ral.close()
        al = hs.HsAligner(hidx, p)
        al.set_two_pass(two_pass)
        got, gctr = al.align(rb, reflib.RESULT_DTYPE, reflib.N_COUNTERS)
        assert differing(want, got) == [], (opt, name, two_pass)
        g = reflib.counters_dict(gctr)
        for k in ("totalReads", "singleHits", "multiHits", "notFound", "nHashTableLookups", "lvCalls", "affineGapCalls", "mapqHistogram"):
            assert wctr[k] == g[k], (opt, name, two_pass, k)
        n_ag += wctr["affineGapCalls"]
    assert n_ag > 100


@pytest.mark.parametrize("opt", list(WHOLE_READ_SCHEMES))
def test_pairs_under_large_scores_match_reference(reflib, small_cfg, opt):
    rp, pp = reflib.default_params_paired(maxDist=27, **WHOLE_READ_SCHEMES[opt]), reflib.default_paired_params()
    ridx, hidx = reflib.RefIndex(small_cfg.idx), hs.HsIndex(small_cfg.idx)
    for name, staged in (("noisy150", False), ("clipped150", True), ("len250", True)):
        pairs = small_cfg.pairs[name]
        want, _ = reflib.RefPairedAligner(ridx, rp, pp).align(pairs)
        al = hs.HsPairedAligner(hidx, rp, pp)
        al.set_staged(staged)
        got, _, _ = al.align(pairs, reflib.PAIRED_RESULT_DTYPE)
        assert differing_pairs(want, got) == [], (opt, name, staged)


@pytest.mark.parametrize("params", [(1, 128, 6, 1), (1, 200, 6, 1), (128, 4, 6, 1), (20, 4, 6, 1), (10, 3999, 3000, 999), (1, 4, 300, 200)])
def test_global_cigar_under_large_scores_equals_reference(reflib, params):
    """sg_ag_cigar.h (the SAM / BAM writer's CIGAR DP) vs AffineGapVectorizedWithCigar::computeGlobalScore under large scores."""
    from test_output_stage import _agc_jobs
    text, pat, qual, jobs = _agc_jobs(reflib, 600, 60 + params[0] + params[1])
    want = reflib.ag_cigar_global_batch(text, pat, qual, jobs, params)
    got = hs.ag_cigar_global_batch(text, pat, qual, jobs, reflib.AGC_OUT_DTYPE, params)
    for f in ("score", "nOps", "netDel", "tailIns"):
        bad = np.nonzero(want[f] != got[f])[0]
        assert bad.size == 0, (f, int(bad[0]), jobs[int(bad[0])], want[int(bad[0])], got[int(bad[0])])
    assert (want["ops"] == got["ops"]).all()
    assert (want["score"] >= 0).mean() > 0.5
