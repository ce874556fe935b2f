#!/usr/bin/env python
"""What `snap paired -ins` costs: paired alignment with and without insert-size inference on bench.py's paired shape (the same
1.5 Gbp synthetic genome, the same seeded 0.5 M-pair batches, stock `snap paired` options) in three forms: device-resident, host
buffers in one call per step, and host buffers in calls of 16384 pairs (the drop-in's default batch of 32768 reads).  The six runs
go in turn, round after round, so that drift on the card falls on all of them alike.  Prints one JSON line with the card's name and
power limit read in the same run, sub-launches per window update and the time of the window statistic.

    python tools/ins_phase.py [--rounds R] [--steps K] [--warmup W] [--genome-mbp 1500] [--batch-reads 1048576] [--call-pairs 16384]

Step times: host clock around each step, which ends in a device synchronise.  The -ins estimator is shared by the steps of a form
(one worker's stream of pairs), with stock's window of 262144 samples, so a 0.5 M-pair step holds about two window updates.
Writes nothing; --json PATH also writes the line to PATH.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    import numpy as np
    import torch
    import bench
    from pass_times import card
    from snap_b200 import engine
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3, help="timed steps per form per round")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--genome-mbp", type=int, default=1500)
    ap.add_argument("--batch-reads", type=int, default=1 << 20)
    ap.add_argument("--batches", type=int, default=2, help="distinct seeded batches the steps cycle through")
    ap.add_argument("--call-pairs", type=int, default=16384, help="pairs per call of the *_host_calls forms (the drop-in's default batch)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    bargs = argparse.Namespace(genome_mbp=args.genome_mbp, batch_reads=args.batch_reads, repeat_frac=0.0, gpus=1)
    c = bench.build_context(bargs)
    batches = bench.make_batches(c, bargs, "paired", args.batches)
    hosts = [bench.to_host_batch(b) for b in batches]
    wl = bench.WORKLOADS["paired"]
    P = args.batch_reads // 2
    al = engine.PairedAligner(c.idx, engine.default_params(**wl["kw"]), engine.default_paired_params(**wl["pkw"]), max_batch_pairs=P)
    est = {"device": engine.SpacingEstimator(al), "host": engine.SpacingEstimator(al), "host_calls": engine.SpacingEstimator(al)}
    stream = torch.cuda.Stream(c.device)
    d_res = torch.empty((P, engine.PAIRED_RESULT_DTYPE.itemsize), dtype=torch.uint8, device=c.device)
    d_ctr = torch.zeros((engine.N_COUNTERS,), dtype=torch.int64, device=c.device)
    h_res = np.zeros(P, dtype=engine.PAIRED_RESULT_DTYPE)

    def step(form, b):
        rb, rq, ro, rl = batches[b % len(batches)][:4]
        hb = hosts[b % len(hosts)]
        if form == "plain_device":
            al.align_device(P, rb.data_ptr(), rq.data_ptr(), ro.data_ptr(), rl.data_ptr(), d_res.data_ptr(), d_ctr.data_ptr(), stream.cuda_stream)
            stream.synchronize()
        elif form == "ins_device":
            est["device"].align_device(P, rb.data_ptr(), rq.data_ptr(), ro.data_ptr(), rl.data_ptr(), d_res.data_ptr(), d_ctr.data_ptr(),
                                       stream.cuda_stream)
            stream.synchronize()
        elif form == "plain_host":
            al.align(hb, out=h_res)
        elif form == "ins_host":
            est["host"].align(hb, out=h_res)
        else:                    # the drop-in's shape: one call per batch of --call-pairs pairs
            for lo in range(0, P, args.call_pairs):
                hi = min(P, lo + args.call_pairs)
                sub = hb.slice(2 * lo, 2 * hi)
                if form == "plain_host_calls":
                    al.align(sub, out=h_res[lo:hi])
                else:
                    est["host_calls"].align(sub, out=h_res[lo:hi])

    forms = ["plain_device", "ins_device", "plain_host", "ins_host", "plain_host_calls", "ins_host_calls"]
    ms = {f: [] for f in forms}
    for f in forms:
        for b in range(args.warmup):
            step(f, b)
    al.check(stream.cuda_stream)
    for r in range(args.rounds):
        for f in forms:
            for k in range(args.steps):
                t0 = time.perf_counter()
                step(f, r * args.steps + k)
                ms[f].append((time.perf_counter() - t0) * 1e3)
    al.check(stream.cuda_stream)
    out = {"workload": wl["cli"] + " [-ins]", "genome_mbp": args.genome_mbp, "pairs_per_step": P, "card": card(), "forms": {}}
    for f in forms:
        v = ms[f]
        out["forms"][f] = {"ms_per_step": {"mean": round(sum(v) / len(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)},
                           "M_reads_per_s": round(2 * P / (sum(v) / len(v)) / 1e3, 3)}
    for where in ("device", "host", "host_calls"):
        st, tm = est[where].get(), est[where].timing()
        plain, ins = out["forms"]["plain_" + where], out["forms"]["ins_" + where]
        out["ins_" + where] = {
            "overhead_vs_plain": round(ins["ms_per_step"]["mean"] / plain["ms_per_step"]["mean"] - 1, 4),
            "updates": st["updates"], "range": [st["minSpacing"], st["maxSpacing"]],
            "sub_launches_per_update": round(tm["subLaunches"] / max(1, st["updates"]), 2),
            "statistic_ms_per_update": round(1e3 * tm["statSeconds"] / max(1, st["updates"]), 3)}
        est[where].close()
    al.close()
    line = json.dumps(out)
    print(line, flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
