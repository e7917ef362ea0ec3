"""Sidecar handle timings on one GPU: cold egs_filter over many 8-GPU nodes for shapes with 3 (one-thread DFS) and
5..8 (leaf-split Trade) branching containers, with the leaves per second that implies, and the steady-state rate of a
sidecar batch.  Records the card name and power limit in the same run.  Writes one JSON object to stdout.

    python tools/sidecar_bench.py [--nodes 10000 100000] [--pods 10000]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import egs_b200  # noqa: E402

SENT = (-1, -1, 0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def cold_filter(n, req, reps):
    e = egs_b200.Egs(0, n, 8, c_max=8)
    e.state_load_bulk(0, 8, 32, np.full((n, 8), 100, np.int32), np.full((n, 8), 32, np.int32))
    e.filter(np.arange(1), req)                              # warm-up: module load, scratch
    e.snapshot()
    ts = []
    for _ in range(reps):
        e.restore()                                          # every option absent again
        t = time.perf_counter(); e.filter(None, req); ts.append(time.perf_counter() - t)
    e.close()
    b = sum(1 for u in req if u[2] == 0)
    s = float(np.median(ts))
    return dict(nodes=n, branching=b, seconds=s, leaves_per_s=n * 8.0 ** b / s)


def steady(n, P):
    """A batch of P sidecar pods of four shapes after every shape's option cache is warm on every node: each pod then
    re-Trades the node the previous pod of its shape was bound to (the leaf-split Trade of one node) and reads the
    cache everywhere else."""
    e = egs_b200.Egs(0, n, 8, c_max=8)
    e.state_load_bulk(0, 8, 32 * 1024, np.full((n, 8), 100, np.int32), np.full((n, 8), 32 * 1024, np.int32))
    rng = np.random.default_rng(1)
    shapes = [[(5 * k + 5, 16 * k + 8, 0)] + [SENT] * (4 + k % 2) for k in range(4)]   # 5 and 6 branching containers
    pods = [shapes[int(rng.integers(0, 4))] for _ in range(P)]
    c_off = np.cumsum([0] + [len(p) for p in pods]).astype(np.int32)
    units = np.array([u for p in pods for u in p], np.int32)
    for sh in shapes:                                        # warm: every shape cached on every node
        e.filter(None, sh)
    t = time.perf_counter(); out = e.schedule_batch(c_off, units); s = time.perf_counter() - t
    e.close()
    return dict(nodes=n, pods=P, seconds=s, decisions_per_s=P / s, bound=int((out["status"] == 0).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, nargs="+", default=[10000, 100000])
    ap.add_argument("--pods", type=int, default=10000)
    ap.add_argument("--max-leaves", type=float, default=float("inf"),
                    help="skip cold-filter workloads whose nodes x leaves exceed this (default: run every workload)")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    shapes = {3: [(10, 4, 0), SENT, SENT, (0, 0, 1), (0, 0, 1)]}
    for b in (5, 6, 7, 8):
        shapes[b] = [(10, 4, 0)] + [SENT] * (b - 1)
    res = dict(card=card(), cold_filter=[], steady=None)
    for n in a.nodes:
        for b, req in shapes.items():
            if n * 8 ** b > a.max_leaves:
                continue
            res["cold_filter"].append(cold_filter(n, req, a.reps))
            print(json.dumps(res["cold_filter"][-1]), file=sys.stderr)
    res["steady"] = steady(a.nodes[0], a.pods)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
