"""Affine-gap scoring schemes (`-gm -gs -go -ge -g5 -g3`) and leaf jobs sized for them, shared by the CPU and GPU scheme tests.

A scheme is given in the reference's order [match, sub, open, extend, 5' bonus, 3' bonus] with the side of sg_ag_small_scores
(snap_b200/csrc/sg_ag.h, at maxReadLen 1000) it is expected to fall on: True = the alignment kernels take the specialised forms
(packed s16x2 rows, narrow-band rows), False = the general int form runs everything."""
from __future__ import annotations

import numpy as np

import jobs as J

# name: (scheme, inside the guard)
SCHEMES = {
    "default": ([1, 4, 6, 1, 10, 7], True),
    "gap_2_5_8_2": ([2, 5, 8, 2, 10, 7], True),
    "sub_eq_open_plus_extend": ([1, 7, 6, 1, 10, 7], True),
    "bonus_0_0": ([1, 4, 6, 1, 0, 0], True),
    "bonus_20_3": ([1, 4, 6, 1, 20, 3], True),
    "gs127": ([1, 127, 6, 1, 10, 7], True),
    "gs128": ([1, 128, 6, 1, 10, 7], True),
    "gs128_go150_ge50": ([1, 128, 150, 50, 10, 7], True),          # gaps dearer than the substitution: the cells take it
    "gs200": ([1, 200, 6, 1, 10, 7], True),
    "gs200_go199": ([1, 200, 199, 1, 10, 7], True),                # sub = open + extend: the largest sub the aligners accept with it
    "gs3999": ([1, 3999, 6, 1, 10, 7], True),
    "go300_ge200": ([1, 4, 300, 200, 10, 7], True),
    "gm127": ([127, 4, 6, 1, 10, 7], False),
    "gm128": ([128, 4, 6, 1, 10, 7], False),
    "gm200": ([200, 4, 6, 1, 10, 7], False),
    "gm20": ([20, 4, 6, 1, 10, 7], False),
    # the guard's edges: top = match * (maxReadLen + MAX_K + 1) + max bonus < 12000, step = max(sub, open + extend) < 4000
    "top_in_step_in": ([10, 3999, 3000, 999, 700, 1], True),       # top 11980, step 3999 (sub and open + extend both at it)
    "step_in_bonus3": ([10, 100, 3900, 99, 1, 700], True),          # step 3999 through open + extend; the larger bonus at the 3' end
    "top_out": ([10, 4, 6, 1, 720, 7], False),                      # top 12000
    "step_out_sub": ([1, 4000, 6, 1, 10, 7], False),
    "step_out_gap": ([1, 4, 3001, 999, 10, 7], False),              # open + extend 4000
    # cells saturate at 32767 on patterns of 170 bases and more: the general form's saturating arithmetic against the reference's
    "saturating": ([100, 4, 6, 1, 10, 7], False),
}

# Bases a job's scoreInit carries from the part of the read before the pattern (default 0: the pattern is the whole read).  At the guard's
# top edge the jobs are tails of 1000-base reads, so that cells come within reach of what the guard admits (above 11 000).
CARRY = {"top_in_step_in": 1128 - 300, "step_in_bonus3": 1128 - 300, "top_out": 1128 - 300}


def scheme_jobs(n: int, seed: int, scheme, carry: int = 0):
    """n jobs in three equal parts: unbanded with patterns of up to 192 columns (the packed form's domain), banded with w <= 15 (the
    narrow-band form's), and wider bands or unbanded patterns of 193..300 columns (the general form's).  scoreInit scales with the
    scheme: mostly between half and all of what a read of the pattern's length (+ carry) can carry (match * length + larger bonus),
    some hopeless ones below that, never above int16."""
    gm, bonus = scheme[0], max(scheme[4], scheme[5])
    parts = []
    for k, max_len in enumerate((192, 150, 300)):
        t, p, q, jb = J.ag_jobs(n // 3, seed * 10 + k, max_len=max_len)
        rng = np.random.default_rng(seed * 10 + k + 5)
        for i in range(jb.size):
            L = int(jb[i]["patternLen"])
            if k == 0:
                jb[i]["banded"] = 0
            elif k == 1:
                wmax = min(15, (L // 3 - 1) // 2)
                if wmax >= 0:
                    jb[i]["w"] = int(rng.integers(0, wmax + 1)) if rng.random() < 0.5 else wmax
                    jb[i]["banded"] = 1
            else:
                wmax = min(63, (L // 3 - 1) // 2)
                if wmax >= 16 and (L <= 192 or rng.random() < 0.5):
                    jb[i]["w"] = int(rng.integers(16, wmax + 1))
                    jb[i]["banded"] = 1
                else:
                    jb[i]["banded"] = 0
            if rng.random() < 0.25:
                # a substitution right at the start (the base next to the seed): the first cells take the substitution penalty
                # itself, with no cheaper gapped path around it
                tc = int(t[int(jb[i]["textOff"]) - (1 if jb[i]["dir"] == -1 else 0)])
                if tc in J.ACGT:
                    p[int(jb[i]["patOff"])] = int(J.ACGT[(list(J.ACGT).index(tc) + int(rng.integers(1, 4))) % 4])
            top = min(gm * (L + carry) + bonus, 32767)
            if rng.random() < 0.85:
                jb[i]["scoreInit"] = int(rng.integers(max(1, top // 2), top + 1))
            else:
                jb[i]["scoreInit"] = int(rng.integers(1, max(2, top // 2)))
        parts.append((t, p, q, jb))
    return _concat(parts)


def _concat(parts):
    """One set of buffers for several (text, pattern, quality, jobs) sets: offsets of the later ones shifted."""
    ts, ps, qs, js = [], [], [], []
    toff = poff = 0
    for t, p, q, jb in parts:
        jb = jb.copy()
        jb["textOff"] += toff
        jb["patOff"] += poff
        ts.append(t); ps.append(p); qs.append(q); js.append(jb)
        toff += t.size
        poff += p.size
    return np.concatenate(ts), np.concatenate(ps), np.concatenate(qs), np.concatenate(js)
