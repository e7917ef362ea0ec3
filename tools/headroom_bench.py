"""egs_headroom on one GPU at config 4 (100 000 nodes x 8 GPUs): the cluster after the first 500 000 pods of config 4,
then the time of one egs_headroom call over every node for config 4's 16 shapes (host clock around the call, which
ends in a device synchronisation; median of --reps calls), and, in the same run, the dry run it replaces for one of
those shapes: egs_checkpoint_save, egs_schedule_batch of the counted total + 1 000 identical pods under EGS_MODE_ROUNDS,
egs_checkpoint_rollback.  The dry run's per-node binds are checked against the headroom counts.  Records the card name
and power limit in the same run.  Writes one JSON object to stdout.

    python tools/headroom_bench.py [--history 500000] [--reps 7] [--dry-shape 0]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import egs_b200  # noqa: E402

ROUNDS = egs_b200.capi.EGS_MODE_ROUNDS


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--history", type=int, default=500_000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--dry-shape", type=int, default=0, help="index into config 4's shapes of the dry-run leg")
    a = ap.parse_args()
    w = egs_b200.workloads.config(4, n_pods=a.history)
    shapes = [list(sh) for sh in egs_b200.workloads.shapes_of(w)]
    e = egs_b200.Egs(w.policy, w.n_nodes, 8)
    e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
    t = time.perf_counter()
    e.schedule_batch(w.c_off, w.units, mode=ROUNDS)
    hist_s = time.perf_counter() - t
    e.headroom(shapes)                                        # warm-up: module load, buffers
    times = []
    for _ in range(a.reps):
        t = time.perf_counter()
        count, failed, summary = e.headroom(shapes)
        times.append(time.perf_counter() - t)
    sh = shapes[a.dry_shape]
    total = int(summary[a.dry_shape, 0] + summary[a.dry_shape, 2])
    K = total + 1000
    c_off = np.arange(K + 1, dtype=np.int32) * len(sh)
    units = np.array(sh * K, np.int32).reshape(-1, 3)
    t = time.perf_counter()
    e.checkpoint_save()
    out = e.schedule_batch(c_off, units, mode=ROUNDS)
    e.checkpoint_rollback()
    dry_s = time.perf_counter() - t
    st, nd = out["status"], out["node"]
    equal = (bool((st[:total] != 1).all() and (st[total:] == 1).all())
             and np.array_equal(np.bincount(nd[st == 0], minlength=w.n_nodes), count[a.dry_shape])
             and np.array_equal(np.bincount(nd[st == 3], minlength=w.n_nodes), failed[a.dry_shape]))
    print(json.dumps(dict(
        card=card(), nodes=w.n_nodes, history_pods=a.history, history_s=round(hist_s, 3), shapes=len(shapes),
        headroom_ms_median=round(1e3 * statistics.median(times), 3), headroom_ms_all=[round(1e3 * x, 3) for x in times],
        summary=summary.tolist(),
        dry_run=dict(shape=sh, pods=K, seconds=round(dry_s, 3), equals_headroom=equal),
    )))


if __name__ == "__main__":
    main()
