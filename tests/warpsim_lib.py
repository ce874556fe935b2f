"""ctypes binding of tests/_build/libwarpsim.so: the TEST-ONLY g++ build of the warp-cooperative device headers
(snap_b200/csrc/sg_warp_ag*.cuh) on the 32-lane SIMT emulator of tests/hostsim/warpsim.h.

Lets the CPU suite run the code the alignment kernels run (shuffles, ballots, DPX s16x2) against the compiled reference.
Never imported by the product package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "_build", "libwarpsim.so")
SRC = os.path.join(HERE, "hostsim", "warpsim.cpp")
CSRC = os.path.join(ROOT, "snap_b200", "csrc")


def build(force: bool = False) -> str:
    deps = [SRC, os.path.join(HERE, "hostsim", "warpsim.h")] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-o", SO, SRC]
    subprocess.run(cmd, check=True)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.ws_ag_batch.restype = C.c_longlong
        L.ws_ag_batch.argtypes = [C.c_void_p] * 5 + [C.c_int64, C.c_void_p, C.c_int]
        L.ws_ag_small_scores.restype = C.c_int
        L.ws_ag_small_scores.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ag_batch(text, pat, qual, jobs, out_dtype, params, packed=1):
    out = np.zeros(jobs.size, dtype=out_dtype)
    params = np.ascontiguousarray(params, dtype=np.int32)
    lib().ws_ag_batch(_p(params), _p(text), _p(pat), _p(qual), _p(np.ascontiguousarray(jobs)), jobs.size, _p(out), packed)
    return out


def small_scores(params) -> bool:
    """sg_ag_small_scores (snap_b200/csrc/sg_ag.h) for a scheme [match, sub, open, extend, 5' bonus, 3' bonus] at maxReadLen 1000 (the
    leaf tests' scratch): True when the kernels may take the specialised affine-gap forms under it."""
    params = np.ascontiguousarray(params, dtype=np.int32)
    return bool(lib().ws_ag_small_scores(_p(params)))
