"""The two-unit narrow-band affine-gap form (snap_b200/csrc/sg_warp_ag_duo.cuh, SgAgParams.usePacked bit 4) on the SIMT emulator of
tests/hostsim/warpsim.h: bit for bit the results of the one-unit form (sg_warp_ag_rows_banded4, usePacked 1) and of the compiled
reference, over every band half-width it takes (0..15), every scoring scheme the kernels run it under, both directions, and the places where its schedule
differs from the one-unit form's: halves that stop their lazy-F loops in different rounds, a half with no unit at the first and last
rows of a call, the row where the band leaves the last segment, and a unit shorter than numVec at the top of the band."""
import functools

import numpy as np
import pytest

import hostsim_lib as hs
import jobs as J
import warpsim_lib as ws
from scheme_jobs import CARRY, SCHEMES, scheme_jobs

ROWS, DUO = 1, 5           # usePacked: packed + one-unit narrow band; + bit 4, the two-unit form


def _banded_sweep(jb, seed):
    """Every job banded, w cycling 0..15 where the pattern allows it (3 (2w + 1) <= patternLen <= 150), both directions."""
    rng = np.random.default_rng(seed)
    keep = []
    for i in range(jb.size):
        L = int(jb[i]["patternLen"])
        wmax = min(15, (L // 3 - 1) // 2)
        if wmax < 0 or L > 150:
            continue
        jb[i]["w"] = min(i % 16, wmax)
        jb[i]["banded"] = 1
        jb[i]["dir"] = 1 if i % 2 else -1
        if rng.random() < 0.2:
            jb[i]["textLen"] = max(1, int(jb[i]["textLen"]) - int(rng.integers(0, 40)))
        keep.append(i)
    return jb[np.array(keep, dtype=np.int64)]


@functools.lru_cache(maxsize=None)
def _scheme_case(name):
    scheme = SCHEMES[name][0]
    t, p, q, jb = scheme_jobs(240, 170 + list(SCHEMES).index(name), scheme, CARRY.get(name, 0))
    return t, p, q, _banded_sweep(jb, 5 + list(SCHEMES).index(name))


@pytest.mark.parametrize("name", [n for n in SCHEMES if SCHEMES[n][1]])
def test_duo_matches_rows_every_scheme(name):
    """Both narrow-band forms run the same cells with the same commit rule, so they agree bit for bit under every scheme the kernels
    run them under (outside sg_ag_small_scores cells can leave int16, and the kernels take the general int form instead)."""
    scheme = SCHEMES[name][0]
    t, p, q, jb = _scheme_case(name)
    assert jb.size > 100 and set(np.unique(jb["dir"])) == {-1, 1}
    a = ws.ag_batch(t, p, q, jb, J.AG_OUT, scheme, ROWS)
    b = ws.ag_batch(t, p, q, jb, J.AG_OUT, scheme, DUO)
    bad = np.nonzero(~J.same_out(a, b))[0]
    assert bad.size == 0, (name, "%d of %d jobs differ" % (bad.size, jb.size), jb[bad[0]], a[bad[0]], b[bad[0]])


@pytest.mark.parametrize("name", [n for n in SCHEMES if SCHEMES[n][1]])
def test_duo_matches_reference_inside_guard(reflib, name):
    """Where the kernels may take the form, against the compiled reference (history-dependent jobs: score and offsets only)."""
    scheme = SCHEMES[name][0]
    t, p, q, jb = _scheme_case(name)
    want = reflib.ag_batch(t, p, q, jb.astype(reflib.AG_JOB_DTYPE), np.array(scheme, dtype=np.int32))
    _, stale = hs.ag_batch(t, p, q, jb, J.AG_OUT, scheme)
    got = ws.ag_batch(t, p, q, jb, J.AG_OUT, scheme, DUO)
    bad = np.nonzero(~J.same_out(want, got) & (stale == 0))[0]
    assert bad.size == 0, (name, jb[bad[0]], want[bad[0]], got[bad[0]])
    for f in ("agScore", "textOffset", "patternOffset"):
        assert (want[f] == got[f]).all(), (name, f)


def _edge_jobs(seed, n, w_of, len_of, text_of, init_of=None):
    t, p, q, jb = J.ag_jobs(n, seed)
    rng = np.random.default_rng(seed)
    keep = []
    for i in range(jb.size):
        L = int(jb[i]["patternLen"])
        w = w_of(i, L, rng)
        if w is None or L < 3 * (2 * w + 1):
            continue
        jb[i]["w"] = w
        jb[i]["banded"] = 1
        jb[i]["patternLen"] = min(L, len_of(i, L, w, rng))
        jb[i]["textLen"] = max(1, min(int(jb[i]["textLen"]), text_of(i, int(jb[i]["patternLen"]), w, rng)))
        if init_of is not None:
            jb[i]["scoreInit"] = init_of(i, int(jb[i]["patternLen"]), rng)
        if int(jb[i]["patternLen"]) >= 3 * (2 * w + 1):
            keep.append(i)
    return t, p, q, jb[np.array(keep, dtype=np.int64)]


def _check(reflib, t, p, q, jb):
    want = reflib.ag_batch(t, p, q, jb.astype(reflib.AG_JOB_DTYPE))
    _, stale = hs.ag_batch(t, p, q, jb, J.AG_OUT, reflib.AG_PARAMS_DEFAULT)
    rows = ws.ag_batch(t, p, q, jb, J.AG_OUT, reflib.AG_PARAMS_DEFAULT, ROWS)
    duo = ws.ag_batch(t, p, q, jb, J.AG_OUT, reflib.AG_PARAMS_DEFAULT, DUO)
    bad = np.nonzero(~J.same_out(rows, duo))[0]
    assert bad.size == 0, (jb[bad[0]], rows[bad[0]], duo[bad[0]])
    bad = np.nonzero(~J.same_out(want, duo) & (stale == 0))[0]
    assert bad.size == 0, (jb[bad[0]], want[bad[0]], duo[bad[0]])


def test_halves_stop_in_different_rounds(reflib):
    """Wide bands (numVec 3 and 4) over patterns with indels, where the two halves' lazy-F loops run for different numbers of rounds;
    and a low scoreInit, under which one half's unit stops at once while the other's F is still alive."""
    t, p, q, jb = _edge_jobs(41, 600, lambda i, L, r: int(r.integers(8, 16)), lambda i, L, w, r: L, lambda i, L, w, r: L + w + 20,
                             lambda i, L, r: (L + 40) if i % 3 else int(r.integers(8, 40)))
    assert jb.size > 200
    _check(reflib, t, p, q, jb)


def test_no_unit_at_first_and_last_row(reflib):
    """Texts of one or two rows (the second half has no unit in the first step, nor the first half in the last) and patterns of one
    segment, where one half never has a unit."""
    t, p, q, jb = _edge_jobs(43, 500, lambda i, L, r: int(r.integers(0, 16)),
                             lambda i, L, w, r: 3 * (2 * w + 1) + int(r.integers(0, 8)) if i % 2 else L,
                             lambda i, L, w, r: int(r.integers(1, 4)) if i % 3 == 0 else L + w)
    assert (jb["textLen"] <= 3).sum() > 50
    _check(reflib, t, p, q, jb)


def test_band_leaves_last_segment(reflib):
    """Texts longer than patternLen + w: the row loop reaches the row whose band starts beyond the last segment (emptyRow)."""
    t, p, q, jb = _edge_jobs(47, 500, lambda i, L, r: int(r.integers(0, 16)), lambda i, L, w, r: L, lambda i, L, w, r: L + w + 40)
    assert ((jb["textLen"] > jb["patternLen"] + jb["w"]) & (jb["dir"] == 1)).sum() > 50
    _check(reflib, t, p, q, jb)


def test_short_unit_at_top_of_band(reflib):
    """Pattern lengths that end a segment part-way (nVecHere < numVec in the last segment's rows) for every w."""
    t, p, q, jb = _edge_jobs(53, 700, lambda i, L, r: i % 16,
                             lambda i, L, w, r: 8 * ((2 * w + 1 + 7) // 8) * int(r.integers(3, 6)) + int(r.integers(1, 8)),
                             lambda i, L, w, r: L + w)
    nv = (2 * jb["w"] + 1 + 7) // 8
    assert ((jb["patternLen"] % (8 * nv)) != 0).sum() > 300
    _check(reflib, t, p, q, jb)
