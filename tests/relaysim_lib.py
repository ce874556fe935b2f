"""ctypes binding of tests/_build/librelaysim.so: the TEST-ONLY host build of what snapgpu_index_save_ex writes (tests/relaysim/relaysim.cpp
over snap_b200/csrc/sg_bucket.h and sg_host.h).  Never imported by the product package."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "_build", "librelaysim.so")
SRC = os.path.join(HERE, "relaysim", "relaysim.cpp")
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
        L.rs_last_error.restype = C.c_char_p
        L.rs_index_open.restype = C.c_void_p
        L.rs_index_open.argtypes = [C.c_char_p, C.c_int]
        L.rs_index_close.argtypes = [C.c_void_p]
        L.rs_write_genome.argtypes = [C.c_void_p, C.c_char_p]
        L.rs_relay_save.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_double]
        _lib = L
    return _lib


class HostIndex:
    """A reference-format index directory loaded on the host (sg_load_index_directory); relayout: switched to sector buckets."""

    def __init__(self, directory: str, relayout: bool = False):
        self.handle = lib().rs_index_open(directory.encode(), 1 if relayout else 0)
        if not self.handle:
            raise RuntimeError(lib().rs_last_error().decode())

    def __del__(self):
        if getattr(self, "handle", None):
            lib().rs_index_close(self.handle)
            self.handle = None

    def write_genome(self, path: str) -> None:
        """Writes the Genome file from the contig lines and bases as loaded (sg_genome_file_header)."""
        if lib().rs_write_genome(self.handle, path.encode()) != 0:
            raise RuntimeError(lib().rs_last_error().decode())

    def relay_save(self, directory: str, key_bytes: int, large: bool = False, slack: float = 0.3) -> None:
        """Writes the bucket-layout index as a reference-format directory in the given table geometry (the host form of
        snapgpu_index_save_ex)."""
        os.makedirs(directory, exist_ok=True)
        if lib().rs_relay_save(self.handle, directory.encode(), key_bytes, 1 if large else 0, slack) != 0:
            raise RuntimeError(lib().rs_last_error().decode())
