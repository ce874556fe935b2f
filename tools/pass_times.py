#!/usr/bin/env python
"""Per-launch times of one `snap single -d 14` step on the headline workload of bench.py (same genome, same seeded reads, same
batch size): the first pass (sg_align_kernel<., 1>), the second (affine-gap) pass (sg_align_kernel<., 2>), the whole step, and the
number of reads the first pass deferred to the second.  Prints one JSON line, with the card's name and power limit read in the same run.

    python tools/pass_times.py [--steps K] [--warmup W] [--pass1-blocks 8,6,5] [--ag-narrow rows,duo,rows,duo]

Kernel times come from torch.profiler (CUDA activities) over K steps; the step time from CUDA events over K other steps, with the
profiler off.  --pass1-blocks runs the steps once per value of SNAPGPU_PASS1_BLOCKS_PER_SM (first-pass CTAs of 8 warps per SM);
--ag-narrow once per value of SNAPGPU_SINGLE_AG_NARROW (the second pass's narrow-band affine-gap form), in the order given, so that
repeating the values alternates them.
Writes nothing; --json PATH also writes the line to PATH.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:          # the times are still worth having; say why the card is unknown
        return {"name": None, "error": str(e)}


def measure(c, args, batches, pass1_blocks, ag_narrow=""):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from snap_b200 import engine
    import bench
    if pass1_blocks:
        os.environ["SNAPGPU_PASS1_BLOCKS_PER_SM"] = str(pass1_blocks)
    else:
        os.environ.pop("SNAPGPU_PASS1_BLOCKS_PER_SM", None)
    if ag_narrow:
        os.environ["SNAPGPU_SINGLE_AG_NARROW"] = ag_narrow
    else:
        os.environ.pop("SNAPGPU_SINGLE_AG_NARROW", None)
    B = args.batch_reads
    al = engine.SingleAligner(c.idx, engine.default_params(**bench.WORKLOADS["single"]["kw"]), max_batch_reads=B)
    stream = torch.cuda.Stream(c.device)
    res = torch.empty((B, engine.RESULT_DTYPE.itemsize), dtype=torch.uint8, device=c.device)
    d_ctr = torch.zeros((engine.N_COUNTERS,), dtype=torch.int64, device=c.device)

    def step(b):
        rb, rq, ro, rl = batches[b % len(batches)][:4]
        al.align_device(B, rb.data_ptr(), rq.data_ptr(), ro.data_ptr(), rl.data_ptr(), res.data_ptr(), d_ctr.data_ptr(), stream.cuda_stream)

    for b in range(args.warmup):
        step(b)
    torch.cuda.synchronize()
    deferred = []
    for b in range(len(batches)):            # the deferred count of each distinct batch (a read defers or not whatever the launch)
        step(b)
        deferred.append(al.deferred_count())
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    ev[0].record(stream)
    for k in range(args.steps):
        step(k)
        ev[k + 1].record(stream)
    torch.cuda.synchronize()
    step_ms = [ev[k].elapsed_time(ev[k + 1]) for k in range(args.steps)]

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for k in range(args.steps):
            step(k)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if not e.name.startswith("void sg_align_kernel<"):
            continue
        m = re.match(r"void sg_align_kernel<(\d+), (\d+)>", e.name)
        key = "pass%s" % m.group(2) if m.group(2) in ("1", "2") else "one_pass"
        d = per.setdefault(key, {"kernel": "sg_align_kernel<%s, %s>" % (m.group(1), m.group(2)), "ms": []})
        d["ms"].append(e.time_range.elapsed_us() / 1e3)
    al.close()
    out = {"pass1_blocks_per_sm": pass1_blocks or "default", "ag_narrow": ag_narrow or "default", "reads_per_step": B, "deferred_reads_per_step": deferred,
           "step_ms": {"mean": round(sum(step_ms) / len(step_ms), 3), "min": round(min(step_ms), 3), "max": round(max(step_ms), 3)}}
    for key, d in sorted(per.items()):
        ms = d["ms"]
        out[key] = {"kernel": d["kernel"], "launches": len(ms), "mean_ms": round(sum(ms) / len(ms), 3), "min_ms": round(min(ms), 3),
                    "max_ms": round(max(ms), 3)}
    if "pass1" in out and "pass2" in out:
        out["pass1_share_of_kernels"] = round(out["pass1"]["mean_ms"] / (out["pass1"]["mean_ms"] + out["pass2"]["mean_ms"]), 4)
    return out


def main():
    import bench
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--genome-mbp", type=int, default=1500)
    ap.add_argument("--batch-reads", type=int, default=1 << 20)
    ap.add_argument("--batches", type=int, default=3, help="distinct seeded batches the steps cycle through")
    ap.add_argument("--pass1-blocks", default="", help="comma-separated SNAPGPU_PASS1_BLOCKS_PER_SM values to sweep (default: the library's own)")
    ap.add_argument("--ag-narrow", default="", help="comma-separated SNAPGPU_SINGLE_AG_NARROW values (rows, duo) to run in turn")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    bargs = argparse.Namespace(genome_mbp=args.genome_mbp, batch_reads=args.batch_reads, repeat_frac=0.0, gpus=1)
    c = bench.build_context(bargs)
    batches = bench.make_batches(c, bargs, "single", args.batches)
    runs = [measure(c, args, batches, int(v) if v else 0, n) for v in (args.pass1_blocks.split(",") if args.pass1_blocks else [""])
            for n in (args.ag_narrow.split(",") if args.ag_narrow else [""])]
    line = json.dumps({"workload": bench.WORKLOADS["single"]["cli"], "genome_mbp": args.genome_mbp, "card": card(),
                       "library": os.environ.get("SNAPGPU_LIB") or "snap_b200/csrc/libsnapgpu.so", "runs": runs})
    print(line, flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
