#!/usr/bin/env python
"""wide_bench.py -- speed of a wide handle (g_max = 16: 16-wide rows, u16 masks, the per-pod batch engine).

  decisions : pod-placement decisions/s of egs_schedule_batch (EGS_MODE_AUTO == the per-pod engine on a wide
              handle) on a 16-GPU cluster: --nodes x 16 GPUs, --pods config-4 pods (core+memory, binpack).  The
              16-GPU rows are config 4's 8-GPU rows side by side (node i = nodes 2i and 2i+1 of config 4), so the
              free-resource distribution is config 4's.  Host clock around the call, which ends in a device sync.
  evaluate  : k_evaluate<16> (the full-evaluate kernel, every node Traded) over --eval-nodes nodes, CUDA-event timed
              with the L2 flushed before each launch, against the N * (8*16 + 5 + 2*C) bytes it has to move:
              16-wide rows (core + mem), fit u8 + score i32, and C u16 masks.

Reads the card's name and power limit in the same run and prints one JSON line (also written to --out).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet (700 W card)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def wide_rows(n_nodes):
    """Config 4's cluster with two 8-GPU nodes joined into one 16-GPU node."""
    import egs_b200
    w = egs_b200.workloads.config(4, n_nodes=2 * n_nodes, n_pods=1)
    return w, w.core.reshape(n_nodes, 16), w.mem.reshape(n_nodes, 16)


def decisions(args):
    import egs_b200
    w8, core, mem = wide_rows(args.nodes)
    pods = egs_b200.workloads.config(4, n_nodes=2, n_pods=args.pods)
    e = egs_b200.Egs(w8.policy, args.nodes, 16)
    e.state_load_bulk(0, 16, w8.mem_total, core, mem)
    e.snapshot()
    warm = pods.prefix(min(args.pods, 2000))
    e.schedule_batch(warm.c_off, warm.units)
    times, placed = [], 0
    for _ in range(args.steps):
        e.restore()
        t0 = time.perf_counter()
        out = e.schedule_batch(pods.c_off, pods.units)       # returns after the device finished (host outputs)
        times.append(time.perf_counter() - t0)
        placed = int((out["status"] == 0).sum())
    e.close()
    med = statistics.median(times)
    return dict(nodes=args.nodes, gpus_per_node=16, pods=args.pods, placed=placed, steps=args.steps,
                seconds_median=med, seconds_min=min(times), seconds_max=max(times),
                decisions_per_s=args.pods / med)


def evaluate(args):
    import egs_b200
    n = args.eval_nodes
    w8, core, mem = wide_rows(n)
    e = egs_b200.Egs(w8.policy, n, 16)
    e.state_load_bulk(0, 16, w8.mem_total, core, mem)
    req = [(20, 4096, 0)]
    e.profile_evaluate(req, iters=3, flush_l2=True)          # warm-up: module load, first touch
    ms = e.profile_evaluate(req, iters=args.eval_iters, flush_l2=True)
    e.close()
    C = len(req)
    nbytes = n * (8 * 16 + 5 + 2 * C)
    bw = nbytes / (ms * 1e-3)
    return dict(nodes=n, containers=C, bytes=nbytes, ms_per_launch=ms, bytes_per_s=bw,
                share_of_hbm_datasheet=bw / HBM_BYTES_PER_S)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000)
    ap.add_argument("--pods", type=int, default=100_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--eval-nodes", type=int, default=2 * 1024 * 1024)
    ap.add_argument("--eval-iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    res = dict(metric="wide_handle", card=card(), decisions=decisions(args), evaluate=evaluate(args))
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
