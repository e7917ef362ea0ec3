#!/usr/bin/env python
"""checkpoint_bench.py -- cost of egs_checkpoint_save / egs_checkpoint_rollback on a config-4 handle (100 000 nodes x
8 GPUs, binpack) after a batch of --pods config-4 pods with library-assigned uids.

  bytes      : what one save (and one rollback) copies on the device: rows (core + mem, 8-wide), mem_total and the
               option tables (state u8, score i32, 4 u8 masks per node) of every interned shape.
  save       : host clock around egs_checkpoint_save plus a synchronise of the handle's stream.
  rollback   : the same around egs_checkpoint_rollback, after an empty what-if and after an 8-pod group.
  device     : the same byte count copied device-to-device by cudaMemcpyAsync (torch), CUDA-event timed: the device
               part of each call.  host = total - device is the rest: the host vectors and the PodBook journal.
  book_pods  : the same calls on a handle whose book holds only a --small-pods batch, so the host part can be
               compared between a book of 10^6 pods and a small one.

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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in q.split(",")]
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def timed(stream, fn):
    t0 = time.perf_counter()
    fn()
    stream.synchronize()
    return time.perf_counter() - t0


def copy_ms(torch, nbytes, iters=20):
    """cudaMemcpyAsync device-to-device of nbytes, CUDA-event timed."""
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda"); b = torch.empty_like(a)
    b.copy_(a); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(iters):
        e0.record(); b.copy_(a); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


def measure(args, n_pods):
    import torch
    import egs_b200
    w = egs_b200.workloads.config(4, n_pods=n_pods)
    e = egs_b200.Egs(w.policy, w.n_nodes, 8)
    e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
    out = e.schedule_batch(w.c_off, w.units)                    # library uids: one run of n_pods in the book
    n_shapes = len(egs_b200.workloads.shapes_of(w))
    stream = torch.cuda.ExternalStream(e.stream_ptr())
    group = w.prefix(8)
    save, rb_empty, rb_group = [], [], []
    for _ in range(args.steps):
        save.append(timed(stream, e.checkpoint_save))
        rb_empty.append(timed(stream, e.checkpoint_rollback))
        e.schedule_batch(group.c_off, group.units)
        rb_group.append(timed(stream, e.checkpoint_rollback))
    e.checkpoint_drop()
    e.close()
    med = lambda xs: statistics.median(xs) * 1e3
    return dict(pods_in_book=n_pods, placed=int((out["status"] == 0).sum()), shapes=n_shapes, steps=args.steps,
                save_ms=med(save), rollback_empty_ms=med(rb_empty), rollback_group8_ms=med(rb_group),
                save_ms_min=min(save) * 1e3, rollback_group8_ms_min=min(rb_group) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=1_000_000)
    ap.add_argument("--small-pods", type=int, default=1_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    import torch
    res = dict(metric="checkpoint", card=card())
    big = measure(args, args.pods)
    small = measure(args, args.small_pods)
    n_pad = (100_000 + 1023) // 1024 * 1024
    rows = n_pad * 8 * 4 * 2 + n_pad * 4
    tables = big["shapes"] * n_pad * (1 + 4 + 4)
    dev = copy_ms(torch, rows + tables)
    res.update(bytes_each_way=rows + tables, bytes_rows=rows, bytes_tables=tables, device_copy_ms=dev)
    for r in (big, small):
        r["save_host_ms"] = r["save_ms"] - dev
        r["rollback_empty_host_ms"] = r["rollback_empty_ms"] - dev
        r["rollback_group8_host_ms"] = r["rollback_group8_ms"] - dev
    res.update(book_1e6=big, book_small=small, card_after=card())
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
