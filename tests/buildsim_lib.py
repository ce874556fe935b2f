"""ctypes binding of tests/_build/libbuildsim.so: the TEST-ONLY host build of what the device index build and save rest on when they
run in passes (tests/buildsim/buildsim.cpp over snap_b200/csrc/sg_bucket.h and sg_host.h).  Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "_build", "libbuildsim.so")
SRC = os.path.join(HERE, "buildsim", "buildsim.cpp")
CSRC = os.path.join(ROOT, "snap_b200", "csrc")


def build(force: bool = False) -> str:
    deps = [SRC] + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".h")]
    if not force and os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return SO
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", SO, SRC], check=True)
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(build())
        L.bs_last_error.restype = C.c_char_p
        L.bs_index_open.restype = C.c_void_p
        L.bs_index_open.argtypes = [C.c_char_p]
        L.bs_index_close.argtypes = [C.c_void_p]
        L.bs_index_relayout.argtypes = [C.c_void_p, C.c_double]
        L.bs_index_buckets_to_tables.argtypes = [C.c_void_p]
        L.bs_index_table_used.restype = C.c_int64
        L.bs_index_table_used.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        L.bs_lookup_seeds.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_uint32, C.c_void_p, C.c_void_p]
        L.bs_bucket_count_for.restype = C.c_uint64
        L.bs_bucket_count_for.argtypes = [C.c_uint64, C.c_uint32, C.c_double]
        L.bs_bucket_min_count.restype = C.c_uint64
        L.bs_bucket_min_count.argtypes = [C.c_uint32]
        L.bs_bucket_mix.restype = C.c_uint64
        L.bs_bucket_mix.argtypes = [C.c_uint64, C.c_uint32]
        L.bs_bucket_unmix.restype = C.c_uint64
        L.bs_bucket_unmix.argtypes = [C.c_uint64, C.c_uint32]
        L.bs_bucket_insert_seq.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32]
        L.bs_bucket_decode.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        L.bs_plan_passes.restype = C.c_int64
        L.bs_plan_passes.argtypes = [C.c_void_p, C.c_uint32, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class BsIndex:
    """A reference-format index directory loaded on the host (sg_load_index_directory)."""

    def __init__(self, directory: str):
        self.handle = lib().bs_index_open(directory.encode())
        if not self.handle:
            raise RuntimeError(lib().bs_last_error().decode())

    def __del__(self):
        if getattr(self, "handle", None):
            lib().bs_index_close(self.handle)
            self.handle = None

    def relayout(self, load: float = 0.0) -> "BsIndex":
        """Switches to the sector-bucket layout (sg_host_relayout)."""
        if lib().bs_index_relayout(self.handle, load) != 0:
            raise RuntimeError(lib().bs_last_error().decode())
        return self

    def buckets_to_tables(self) -> "BsIndex":
        """Switches a bucket-layout index back to the reference's tables, re-laid from the buckets (sg_host_buckets_to_tables)."""
        if lib().bs_index_buckets_to_tables(self.handle) != 0:
            raise RuntimeError(lib().bs_last_error().decode())
        return self

    def table_used(self) -> np.ndarray:
        """Used entries per table: as the directory's table headers state them, or as the last re-lay into tables counted them."""
        n = lib().bs_index_table_used(self.handle, None, 0)
        out = np.zeros(n, dtype=np.uint64)
        lib().bs_index_table_used(self.handle, _p(out), n)
        return out

    def lookup(self, seeds: np.ndarray, n: int, max_hits: int = 512):
        nh = np.zeros(2 * n, dtype=np.int64)
        hits = np.zeros(2 * n * max_hits, dtype=np.uint32)
        lib().bs_lookup_seeds(self.handle, _p(seeds), n, max_hits, _p(nh), _p(hits))
        return nh.reshape(n, 2), hits.reshape(n, 2, max_hits)


def bucket_count_for(n_entries: int, seed_len: int, load: float) -> int:
    return int(lib().bs_bucket_count_for(n_entries, seed_len, load))


def bucket_min_count(bits: int) -> int:
    return int(lib().bs_bucket_min_count(bits))


def bucket_mix(c: int, bits: int) -> int:
    return int(lib().bs_bucket_mix(c, bits))


def bucket_unmix(h: int, bits: int) -> int:
    return int(lib().bs_bucket_unmix(h, bits))


def bucket_image(n_buckets: int) -> np.ndarray:
    """An empty sector-bucket image (every slot SG_BUCKET_EMPTY)."""
    return np.full(n_buckets * 4, 0x3fffffffffffffff, dtype=np.uint64)


def bucket_insert_seq(buckets: np.ndarray, n_buckets: int, bits: int, canonical: int, orient: int, value: int) -> bool:
    return lib().bs_bucket_insert_seq(_p(buckets), n_buckets, bits, canonical, orient, value) == 1


def bucket_decode(buckets: np.ndarray, n_buckets: int, seed_len: int, slots: np.ndarray):
    """(seed, orientation) of the given slots through sg_bucket_slot_decode; orientation 255 where it fails."""
    idx = np.ascontiguousarray(slots, dtype=np.uint64)
    seeds = np.zeros(idx.size, dtype=np.uint64)
    orients = np.zeros(idx.size, dtype=np.uint8)
    lib().bs_bucket_decode(_p(buckets), n_buckets, seed_len, _p(idx), idx.size, _p(seeds), _p(orients))
    return seeds, orients


def plan_passes(bin_bytes, budget: int, min_passes: int = 1):
    """sg_plan_passes: the pass edges (P + 1 of them), or (None, bad bin) when one bin exceeds the budget."""
    b = np.ascontiguousarray(bin_bytes, dtype=np.uint64)
    bounds = np.zeros(b.size + 1, dtype=np.uint32)
    bad = C.c_uint32(0)
    p = lib().bs_plan_passes(_p(b), b.size, budget, min_passes, _p(bounds), C.byref(bad))
    if p < 0:
        return None, int(bad.value)
    return bounds[:p + 1].astype(np.int64), None
