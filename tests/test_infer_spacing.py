"""Insert-size inference (`snap paired -ins`) on the host: the window statistic of snap_b200/csrc/sg_spacing.h against the
reference's own PairedAlignerContext::computeSpacingDist, and its per-pair sample rule against a restatement of
PairedAligner.cpp:822-925.  No GPU."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
W = 262144
INVALID = 0xFFFFFFFF


@pytest.fixture(scope="module")
def libs(tmp_path_factory, reflib):
    d = tmp_path_factory.mktemp("spacing")
    host = str(d / "libhostspacing.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", host,
                    os.path.join(HERE, "spacing", "host_spacing.cpp")], check=True)
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    ref = str(d / "librefspacing.so")
    # the reference's own flags (oracle/Makefile)
    subprocess.run(["g++", "-O3", "-Wno-format", "-std=c++98", "-msse", "-fPIC", "-w", "-I" + os.path.join(ref_dir, "include"), "-shared",
                    "-o", ref, os.path.join(HERE, "spacing", "ref_spacing.cpp"), "-L" + ref_dir, "-lsnapref", "-Wl,-rpath," + ref_dir],
                   check=True)
    H, R = C.CDLL(host), C.CDLL(ref)
    H.host_spacing_range.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    H.host_spacing_samples.argtypes = [C.c_int64, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    R.ref_compute_spacing_dist.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    return H, R


def _windows():
    rng = np.random.default_rng(2024)
    out = {}
    for k in range(5):
        out["normal%d" % k] = rng.normal(300 + 40 * k, 30 + 5 * k, W).round().clip(0)
    for k in range(5):
        n1 = int(W * (0.85 - 0.05 * k))
        out["bimodal%d" % k] = np.concatenate([rng.normal(300, 30, n1), rng.normal(800, 60, W - n1)]).round().clip(0)
    for k, v in enumerate([0, 1, 500, INVALID]):
        out["equal%d" % k] = np.full(W, v)
    for k in range(4):
        out["near0_%d" % k] = rng.integers(0, 3 + 4 * k, W)
    for k, frac in enumerate([0.0005, 0.01, 0.1, 0.2]):
        a = rng.normal(350, 40, W).round().clip(0)
        a[rng.random(W) < frac] = INVALID
        out["fewinvalid%d" % k] = a
    for k, frac in enumerate([0.26, 0.3, 0.5, 0.8]):
        a = rng.normal(350, 40, W).round().clip(0)
        a[rng.random(W) < frac] = INVALID
        out["manyinvalid%d" % k] = a
    for k, frac in enumerate([0.3, 0.6]):        # NotFound beside a located end: distance = InvalidGenomeLocation - location
        a = rng.normal(350, 40, W).round().clip(0)
        m = rng.random(W) < frac
        a[m] = INVALID - rng.integers(0, 3_000_000_000, int(m.sum()))
        out["halfinvalid%d" % k] = a
    out["uniform_wide"] = rng.integers(0, 1 << 33, W)
    out["lognormal"] = rng.lognormal(6, 1.5, W).round()
    out["exp_small"] = rng.exponential(3, W).round()
    return {k: np.sort(np.asarray(v, dtype=np.int64)) for k, v in out.items()}


def test_window_statistic_matches_reference(libs):
    H, R = libs
    wins = _windows()
    assert len(wins) >= 30
    seen = set()
    for name, s in wins.items():
        s = np.ascontiguousarray(s)
        rmn, rmx, hmn, hmx = C.c_int(), C.c_int(), C.c_int32(), C.c_int32()
        R.ref_compute_spacing_dist(s.ctypes.data, C.byref(rmn), C.byref(rmx))
        H.host_spacing_range(s.ctypes.data, W, C.byref(hmn), C.byref(hmx))
        assert (hmn.value, hmx.value) == (rmn.value, rmx.value), name
        seen.add((rmn.value == 1, rmx.value == -2**31 or rmn.value == -2**31))
    # the clamp to 1 and the out-of-range conversion both occur
    assert any(a for a, _ in seen) and any(b for _, b in seen)


def test_bimodal_window_gives_the_documented_range(libs):
    """85 % N(300, 30) + 15 % N(800, 60): s25 ~ 283, s75 ~ 335, and the IQR x 3 bounds are the range (about 130..490)."""
    H, _ = libs
    rng = np.random.default_rng(7)
    n1 = int(0.85 * W)
    s = np.sort(np.concatenate([rng.normal(300, 30, n1), rng.normal(800, 60, W - n1)]).round().astype(np.int64))
    mn, mx = C.c_int32(), C.c_int32()
    H.host_spacing_range(s.ctypes.data, W, C.byref(mn), C.byref(mx))
    assert 100 < mn.value < 160 and 460 < mx.value < 520


def _py_sample(st, dr, loc, useful, flags, force):
    """PairedAligner.cpp:822-925 for one pair: the sample it adds to the window, or -1."""
    if not useful[0] and not useful[1]:
        return -1
    st, loc = list(st), list(loc)
    if force and (st[0] == 1) != (st[1] == 1):
        st = [0, 0]
        loc = [INVALID, INVALID]

    def pass_filter(status, too_short):
        if flags == 0:
            return True
        if too_short:
            return bool(flags & 0x10)
        return bool(flags & {0: 0x1, 1: 0x2, 2: 0x4}[status])
    p0, p1 = pass_filter(st[0], not useful[0]), pass_filter(st[1], not useful[1])
    primary = (p0 and p1) if flags & 0x8 else (p0 or p1)
    if not primary or dr[0] == dr[1]:
        return -1
    return abs(loc[0] - loc[1])


@pytest.mark.parametrize("flags,force", [(0, 0), (0x16, 1), (0x16 | 0x8, 0), (0x11, 0), (0x3, 1), (0x1c, 0)])
def test_sample_rule_matches_restatement(libs, flags, force):
    from oracle import reflib
    H, _ = libs
    rng = np.random.default_rng(flags * 2 + force)
    n = 20000
    r = np.zeros(n, dtype=reflib.PAIRED_RESULT_DTYPE)
    r["status"] = rng.integers(0, 3, (n, 2))
    r["direction"] = rng.integers(0, 2, (n, 2))
    loc = rng.integers(0, 1 << 31, (n, 2))
    loc[r["status"] == 0] = INVALID
    near = rng.random(n) < 0.5
    loc[near, 1] = loc[near, 0] + rng.integers(-1000, 1000, int(near.sum()))
    r["location"] = loc
    useful = (rng.random((n, 2)) < 0.9).astype(np.uint8)
    got = np.zeros(n, dtype=np.int64)
    H.host_spacing_samples(n, r.ctypes.data, useful.ctypes.data, flags, force, got.ctypes.data)
    want = [_py_sample(r["status"][i], r["direction"][i], [int(x) for x in r["location"][i]], useful[i], flags, force) for i in range(n)]
    assert got.tolist() == want
    assert (got >= 0).sum() > n // 20


# ---- rule and schedule: the host build of the aligner and of sg_spacing.h against the reference aligner, at a window of 1000 ----

WIN = 1000
OPTION_SETS = {                 # (params, paired params, filterFlags): default, `-fs -F a`, `-F a -F b`
    "default": (dict(maxDist=14), dict(), 0),
    "fs_Fa": (dict(maxDist=14), dict(forceSpacing=1), 0x16),
    "Fa_Fb": (dict(maxDist=14), dict(), 0x16 | 0x8),
}


def _py_range(s):
    """computeSpacingDist (PairedAligner.cpp:424-458) over a sorted window of any size, in Python doubles."""
    import math
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


def _drive(pb, n, align, samples_of, range_of, mn, mx, chunk=1200):
    """PairedAligner.cpp:889-925 over pairs [0, n): align(lo, hi, mn, mx) -> results of pairs [lo, hi) under (mn, mx);
    samples_of(results, lo) -> each pair's sample or -1; range_of(sorted window) -> (mn, mx).  Returns (results, updates) with
    updates = [(first pair under the new range, mn, mx)]."""
    out, updates, win, p = None, [], [], 0
    while p < n:
        hi = min(n, p + chunk)
        res = align(p, hi, mn, mx)
        if out is None:
            out = np.zeros(n, dtype=res.dtype)
        smp = samples_of(res, p)
        j = p
        while j < hi:
            out[j] = res[j - p]
            j += 1
            if smp[j - 1 - p] >= 0:
                win.append(int(smp[j - 1 - p]))
                if len(win) == WIN:
                    mn, mx = range_of(sorted(win))
                    mx &= 0xFFFFFFFF                 # setMaxSpacing(int) into an unsigned
                    win = []
                    updates.append((j, mn, mx))
                    break
        p = j
    return out, updates


@pytest.fixture(scope="module")
def ins_cfg(tmp_path_factory, reflib):
    from snap_b200 import synth
    d = tmp_path_factory.mktemp("insref")
    contigs = synth.make_contigs(3, 200_000, seed=91, repeat_frac=0.1)
    synth.write_fasta(str(d / "ref.fa"), contigs)
    reflib.build_reference_index(reflib.SNAP_ALIGNER, str(d / "ref.fa"), str(d / "idx"))
    n = 6000
    n2 = int(0.15 * n)          # ~85 % N(300, 30) and 15 % N(800, 60) inserts, in random order
    a = synth.make_pairs(contigs, n - n2, 100, seed=17, insert_mean=300, insert_sd=30, chimeric_frac=0.02, n_run_frac=0.02, short_frac=0.02)
    b = synth.make_pairs(contigs, n2, 100, seed=18, insert_mean=800, insert_sd=60)
    reads = []
    for j in np.random.default_rng(17).permutation(n):
        src, i = (a, j) if j < n - n2 else (b, j - (n - n2))
        reads += [src.read(2 * i), src.read(2 * i + 1)]
    return str(d / "idx"), synth.ReadBatch.from_lists(reads)


@pytest.mark.parametrize("opt", list(OPTION_SETS))
def test_rule_and_schedule_match_the_reference_aligner(libs, reflib, ins_cfg, opt):
    import hostsim_lib as hs
    from conftest import differing_pairs
    H, _ = libs
    idx, pb = ins_cfg
    n = pb.n // 2
    kw, pkw, flags = OPTION_SETS[opt]
    force = pkw.get("forceSpacing", 0)
    useful = np.array([pb.lens[i] >= 50 and pb.read(i)[0].count(b"N") <= kw["maxDist"] for i in range(pb.n)], dtype=np.uint8)
    mn0, mx0 = 0, 1000
    ridx, hidx = reflib.RefIndex(idx), hs.HsIndex(idx)

    def ref_align(lo, hi, mn, mx):
        ral = reflib.RefPairedAligner(ridx, reflib.default_params_paired(**kw), reflib.default_paired_params(**{**pkw, "minSpacing": mn, "maxSpacing": mx}))
        res, _ = ral.align(pb.slice(2 * lo, 2 * hi))
        ral.close()
        return res

    def ref_samples(res, lo):
        return [_py_sample(res["status"][k], res["direction"][k], [int(x) for x in res["location"][k]], useful[2 * (lo + k):2 * (lo + k) + 2], flags, force)
                for k in range(len(res))]

    def host_align(lo, hi, mn, mx):
        hal = hs.HsPairedAligner(hidx, reflib.default_params_paired(**kw), reflib.default_paired_params(**{**pkw, "minSpacing": mn, "maxSpacing": mx}))
        res, _, _ = hal.align(pb.slice(2 * lo, 2 * hi), reflib.PAIRED_RESULT_DTYPE)
        return res

    def host_samples(res, lo):
        res = np.ascontiguousarray(res)
        u = np.ascontiguousarray(useful[2 * lo:2 * lo + 2 * len(res)])
        out = np.zeros(len(res), dtype=np.int64)
        H.host_spacing_samples(len(res), res.ctypes.data, u.ctypes.data, flags, force, out.ctypes.data)
        return out

    def host_range(s):
        a = np.array(s, dtype=np.int64)
        mn, mx = C.c_int32(), C.c_int32()
        H.host_spacing_range(a.ctypes.data, len(a), C.byref(mn), C.byref(mx))
        return mn.value, mx.value

    want, want_upd = _drive(pb, n, ref_align, ref_samples, _py_range, mn0, mx0)
    got, got_upd = _drive(pb, n, host_align, host_samples, host_range, mn0, mx0)
    assert len(want_upd) >= 4, want_upd
    # the long-insert population (end-to-end distance ~700) leaves the intersecting aligner after the first update
    assert all(1 <= mn and mx < 600 for _, mn, mx in want_upd), want_upd
    assert got_upd == want_upd
    assert differing_pairs(want, got) == []
