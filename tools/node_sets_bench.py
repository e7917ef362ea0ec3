"""Candidate node sets (egs_schedule_batch_nodes) on one GPU at config 4 (100 000 nodes x 8 GPUs, 1 M pods): decisions
per second and egs_rounds_stats of egs_schedule_batch, one all-ones set, one set of 90 % of the nodes, and two disjoint
half-cluster pools alternating in runs of 10 000 / 1 000 / 100 / 10 pods; then the per-pod engine of a wide
(g_max = 16) and of a sidecar (c_max = 8) handle, with every node and with a 90 % set.  Every leg starts from the
same loaded cluster with cold option caches (egs_state_restore).  Records the card name and power limit in the same
run.  Writes one JSON object to stdout.

    python tools/node_sets_bench.py [--pods 1000000] [--short-pods 100000]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import egs_b200  # noqa: E402

ROUNDS = egs_b200.capi.EGS_MODE_ROUNDS
SENT = (-1, -1, 0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(e, fn, P):
    e.restore()
    s0 = e.rounds_stats()
    t = time.perf_counter(); out = fn(); s = time.perf_counter() - t
    s1 = e.rounds_stats()
    return dict(pods=P, seconds=s, decisions_per_s=P / s, bound=int((out["status"] == 0).sum()),
                rounds_stats={k: int(s1[k] - s0[k]) for k in s1}), out


def config4(P, short_p):
    w = egs_b200.workloads.config(4, n_pods=P)
    N = w.n_nodes
    e = egs_b200.Egs(w.policy, N, 8)
    e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
    e.snapshot()
    warm = w.prefix(10000)
    e.schedule_batch(warm.c_off, warm.units, mode=ROUNDS)
    rng = np.random.default_rng(4)
    ones, ninety = np.ones(N, bool), rng.random(N) < 0.9
    left = np.zeros(N, bool); left[:N // 2] = True
    res = {}
    res["schedule_batch"], ref = timed(e, lambda: e.schedule_batch(w.c_off, w.units, mode=ROUNDS), P)
    res["all_ones"], got = timed(e, lambda: e.schedule_batch_nodes(w.c_off, w.units, [ones], mode=ROUNDS), P)
    res["all_ones"]["outputs_equal_schedule_batch"] = all(np.array_equal(ref[f], got[f]) for f in ref)
    res["ninety_percent"], _ = timed(e, lambda: e.schedule_batch_nodes(w.c_off, w.units, [ninety], mode=ROUNDS), P)
    pools = egs_b200.capi.node_sets_array([left, ~left], N)
    for run in (10000, 1000, 100, 10):
        p = P if run >= 1000 else short_p
        s = w.prefix(p)
        pod_set = (np.arange(p) // run % 2).astype(np.int32)
        key = f"pools_run_{run}"
        res[key], _ = timed(e, lambda: e.schedule_batch_nodes(s.c_off, s.units, pools, pod_set, mode=ROUNDS), p)
        res[key]["runs"] = -(-p // run)
        print(json.dumps({key: res[key]}), file=sys.stderr)
    e.close()
    return res


def per_pod(kind, n, P):
    """The per-pod engine (EGS_MODE_RESCAN) of a wide or a sidecar handle, every node vs a 90 % set."""
    rng = np.random.default_rng(16 if kind == "wide" else 8)
    g = 16 if kind == "wide" else 8
    e = egs_b200.Egs(0, n, g, c_max=8 if kind == "sidecar" else 4)
    e.state_load_bulk(0, g, 80 * 1024, np.full((n, g), 100, np.int32), np.full((n, g), 80 * 1024, np.int32))
    e.snapshot()
    if kind == "wide":
        shapes = [[(20, 4096, 0)], [(0, 0, 1)], [(0, 0, 10)], [(50, 8192, 0), (0, 0, 2)]]
    else:
        shapes = [[(5 * k + 5, 1024 * k + 512, 0)] + [SENT] * (4 + k % 2) for k in range(4)]
    pods = [shapes[int(rng.integers(0, len(shapes)))] for _ in range(P)]
    c_off = np.cumsum([0] + [len(p) for p in pods]).astype(np.int32)
    units = np.array([u for p in pods for u in p], np.int32)
    e.schedule_batch(c_off[:101], units[:c_off[100]])                 # warm-up: module load, scratch
    ninety = rng.random(n) < 0.9
    res = {}
    res["schedule_batch"], _ = timed(e, lambda: e.schedule_batch(c_off, units), P)
    res["ninety_percent"], _ = timed(e, lambda: e.schedule_batch_nodes(c_off, units, [ninety]), P)
    e.close()
    return dict(nodes=n, **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pods", type=int, default=1000000)
    ap.add_argument("--short-pods", type=int, default=100000, help="pods of the legs with runs of 100 and 10")
    ap.add_argument("--per-pod-nodes", type=int, default=10000)
    ap.add_argument("--per-pod-pods", type=int, default=10000)
    a = ap.parse_args()
    res = dict(card=card(), config4=config4(a.pods, a.short_pods))
    for kind in ("wide", "sidecar"):
        res[kind] = per_pod(kind, a.per_pod_nodes, a.per_pod_pods)
        print(json.dumps({kind: res[kind]}), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
