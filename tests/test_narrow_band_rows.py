"""The one-unit narrow-band affine-gap form (snap_b200/csrc/sg_warp_ag.cuh: sg_warp_ag_rows_banded4, SgAgParams.usePacked 1) on the
SIMT emulator of tests/hostsim/warpsim.h, against the compiled reference directly: every band half-width 0..15 (1..4 vectors per
segment), both directions, patterns that end a segment part-way, texts that run past the band's last segment, and low scoreInit."""
import numpy as np
import pytest

import hostsim_lib as hs
import jobs as J
import warpsim_lib as ws

ROWS = 1                   # usePacked: packed + one-unit narrow band


def _jobs(seed, n, len_of, text_of, init_of=None):
    t, p, q, jb = J.ag_jobs(n, seed)
    rng = np.random.default_rng(seed)
    keep = []
    for i in range(jb.size):
        L = int(jb[i]["patternLen"])
        w = i % 16
        jb[i]["w"] = w
        jb[i]["banded"] = 1
        jb[i]["dir"] = 1 if (i // 16) % 2 else -1
        jb[i]["patternLen"] = min(L, len_of(i, L, w, rng))
        jb[i]["textLen"] = max(1, min(int(jb[i]["textLen"]), text_of(i, int(jb[i]["patternLen"]), w, rng)))
        if init_of is not None:
            jb[i]["scoreInit"] = init_of(i, int(jb[i]["patternLen"]), rng)
        if int(jb[i]["patternLen"]) >= 3 * (2 * w + 1):
            keep.append(i)
    return t, p, q, jb[np.array(keep, dtype=np.int64)]


CASES = {
    # whole patterns, texts reaching past patternLen + w
    "plain": (lambda i, L, w, r: L, lambda i, L, w, r: L + w + int(r.integers(0, 40)), None),
    # pattern lengths that end a segment part-way (fewer vectors than numVec in the last segment's rows)
    "short_last_segment": (lambda i, L, w, r: 8 * ((2 * w + 1 + 7) // 8) * int(r.integers(3, 6)) + int(r.integers(1, 8)),
                           lambda i, L, w, r: L + w, None),
    # low scoreInit: rows stop early and hInit of segment 0 falls to 0
    "low_score_init": (lambda i, L, w, r: L, lambda i, L, w, r: L + w, lambda i, L, r: int(r.integers(4, 40))),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_rows_match_reference(reflib, case):
    len_of, text_of, init_of = CASES[case]
    t, p, q, jb = _jobs(61 + sorted(CASES).index(case), 900, len_of, text_of, init_of)
    nv = (np.minimum(2 * jb["w"] + 1, jb["patternLen"]) + 7) // 8
    assert set(np.unique(jb["w"])) == set(range(16)) and set(np.unique(nv)) == {1, 2, 3, 4}
    assert set(np.unique(jb["dir"])) == {-1, 1}
    want = reflib.ag_batch(t, p, q, jb.astype(reflib.AG_JOB_DTYPE))
    _, stale = hs.ag_batch(t, p, q, jb, J.AG_OUT, reflib.AG_PARAMS_DEFAULT)
    got = ws.ag_batch(t, p, q, jb, J.AG_OUT, reflib.AG_PARAMS_DEFAULT, ROWS)
    # jobs whose result depends on cells of earlier calls (stale) agree on score and offsets only
    bad = np.nonzero(~J.same_out(want, got) & (stale == 0))[0]
    assert bad.size == 0, (case, "%d of %d jobs differ" % (bad.size, jb.size), jb[bad[0]], want[bad[0]], got[bad[0]])
    for f in ("agScore", "textOffset", "patternOffset"):
        assert (want[f] == got[f]).all(), (case, f)
