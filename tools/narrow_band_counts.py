#!/usr/bin/env python
"""Counts, on the CPU, what the two narrow-band affine-gap forms of the single-end second pass run on bench.py's headline workload
(`snap single -d 14`, 150 bp reads from bench.py's generator), at a small genome.  Deterministic; no GPU.

    python tools/narrow_band_counts.py [--genome-mbp 24] [--reads 100000]

The genome and reads come from bench.py's generator (snap_b200/synth_device.py) run by torch on the CPU; the index is built by the
reference's `snap index`; the reads go through the host build of the aligner in its two-pass form (tests/hostsim), whose scalar
affine-gap form reports every call and every (row, segment) unit with the lazy-F rounds it entered (tools/narrow_band_counts.cpp).
Only the second pass rescores with affine gap, so every call counted is one the second pass makes.  For the banded calls of up to
4 vectors per segment (w <= 15):
  rows (sg_warp_ag_rows_banded4): one warp step per unit, running that unit's rounds;
  duo  (sg_warp_ag_rows_banded_duo): two units per step (unit (row i, segment j) at step i + j), running the longer of their loops.
Multiply the steps and rounds by the SASS instructions of a step and of a round to predict the instruction counts.  Prints one JSON
line; builds in a temporary directory and writes nothing in the tree.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

N = 48
CALLS, UNITS, ROWS, ROUNDS_ROWS, STEPS_DUO, ROUNDS_DUO, STEPS_ONE_UNIT = range(7)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--genome-mbp", type=int, default=24)
    ap.add_argument("--reads", type=int, default=100_000)
    ap.add_argument("--seed", type=int, default=1000, help="read seed (bench.py's first batch uses 1000)")
    args = ap.parse_args()

    import torch
    import bench
    import hostsim_lib as hs
    from oracle import reflib
    from snap_b200 import synth, synth_device

    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "libnbcounts.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                        os.path.join(ROOT, "tools", "narrow_band_counts.cpp")], check=True)
        hs.build = lambda force=False: so          # hostsim_lib's bindings, on the counting build
        hs._lib = None
        L = hs.lib()
        L.nb_counts.argtypes = [C.c_void_p]

        n_contigs = 24
        contig_len = args.genome_mbp * 1_000_000 // n_contigs
        bases, starts = synth_device.make_genome(n_contigs, contig_len, seed=20260924, device="cpu")
        b = bases.numpy()
        synth.write_fasta(os.path.join(d, "ref.fa"), [b[s:s + contig_len] for s in starts])
        reflib.build_reference_index(reflib.SNAP_ALIGNER, os.path.join(d, "ref.fa"), os.path.join(d, "idx"), seed_len=bench.SEED_LEN)
        rb = bench.to_host_batch(synth_device.make_reads(bases, starts, contig_len, args.reads, bench.READ_LEN, seed=args.seed), pinned=False)

        p = reflib.default_params(**bench.WORKLOADS["single"]["kw"])
        al = hs.HsAligner(hs.HsIndex(os.path.join(d, "idx")), p)
        al.set_two_pass(True)
        L.nb_reset()
        _, ctr = al.align(rb, reflib.RESULT_DTYPE, reflib.N_COUNTERS)
        deferred = al.deferred
        c = np.zeros(N, dtype=np.int64)
        L.nb_counts(c.ctypes.data_as(C.c_void_p))

    units, steps = int(c[UNITS]), int(c[STEPS_DUO])
    out = {
        "workload": bench.WORKLOADS["single"]["cli"], "genome_mbp": args.genome_mbp, "reads": args.reads,
        "deferred_reads": int(deferred), "affine_gap_calls": int(reflib.counters_dict(ctr)["affineGapCalls"]),
        "narrow_calls": int(c[CALLS]), "narrow_rows": int(c[ROWS]),
        "calls_by_numVec": {str(v): int(c[8 + v - 1]) for v in range(1, 5)},
        "units_by_numVec": {str(v): int(c[12 + v - 1]) for v in range(1, 5)},
        "calls_by_w": {str(w): int(c[16 + w]) for w in range(16) if c[16 + w]},
        "units_by_nVecHere": {str(v): int(c[32 + v]) for v in range(5) if c[32 + v]},
        "unit_rounds_hist": {str(r): int(c[40 + r - 1]) for r in range(1, 8)},
        "rows": {"warp_steps": units, "lazy_f_rounds": int(c[ROUNDS_ROWS]),
                 "rounds_per_unit": round(int(c[ROUNDS_ROWS]) / max(units, 1), 3)},
        "duo": {"warp_steps": steps, "steps_with_one_unit": int(c[STEPS_ONE_UNIT]), "lazy_f_rounds": int(c[ROUNDS_DUO]),
                "rounds_per_step": round(int(c[ROUNDS_DUO]) / max(steps, 1), 3)},
    }
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
