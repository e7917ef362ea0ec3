"""egs_evict_fit on one GPU at config 4 (100 000 nodes x 8 GPUs): the cluster after the first 500 000 pods of config 4,
then one eviction what-if over --nodes candidate nodes with 1 to 4 victims each, taken from the pods the batch placed
on them.  Times one egs_evict_fit call (host clock around the C call, which ends in a device synchronisation; its
arguments packed beforehand; median of --reps calls after a warm-up) and, in the same run, the checkpoint sequence it
replaces on --seq-nodes of those nodes: egs_checkpoint_save, egs_pod_cancel of each victim, egs_filter / egs_score /
egs_bind of the pending pod on that node, egs_checkpoint_rollback, reported per node.  The sequence's answers are checked against the call's.  Records the card
name and power limit in the same run.  Writes one JSON object to stdout.

    python tools/evict_bench.py [--history 500000] [--nodes 10000] [--seq-nodes 100] [--reps 7] [--shape K]

The pending pod is config 4's shape K, by default its largest (the one that fits on the fewest nodes)."""
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

cap = egs_b200.capi
ROUNDS = cap.EGS_MODE_ROUNDS


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--history", type=int, default=500_000)
    ap.add_argument("--nodes", type=int, default=10_000)
    ap.add_argument("--seq-nodes", type=int, default=100)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shape", type=int, default=None, help="index into config 4's shapes of the pending pod")
    a = ap.parse_args()
    w = egs_b200.workloads.config(4, n_pods=a.history)
    shapes = [list(sh) for sh in egs_b200.workloads.shapes_of(w)]
    e = egs_b200.Egs(w.policy, w.n_nodes, 8)
    e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
    uids = np.arange(1, a.history + 1, dtype=np.uint64)
    out = e.schedule_batch(w.c_off, w.units, uids, mode=ROUNDS)

    # the placements of the batch, per node
    placed = {}
    for p in np.nonzero(out["status"] == 0)[0]:
        req = [tuple(int(x) for x in w.units[k]) for k in range(w.c_off[p], w.c_off[p + 1])]
        placed.setdefault(int(out["node"][p]), []).append((req, cap.masks_to_lists(out["alloc_mask"][p], len(req)),
                                                           int(uids[p])))
    rng = np.random.default_rng(0)
    ids = rng.permutation(sorted(placed))[:a.nodes].astype(np.int32)
    victims = []
    for n in ids.tolist():
        pods = placed[n]
        k = int(rng.integers(1, 5))
        victims.append([pods[int(i)] for i in rng.choice(len(pods), min(k, len(pods)), replace=False)])
    req = shapes[a.shape] if a.shape is not None else max(shapes, key=lambda sh: (sh[0][1], sh[0][0]))

    # the call's arguments, packed once
    n = len(ids)
    units = cap.units_array(req)
    off = np.concatenate([[0], np.cumsum([len(v) for v in victims])]).astype(np.int32)
    recs = cap.mutations_array([(cap.EGS_MUT_FORGET, int(nd), u, al, uid) for nd, vs in zip(ids.tolist(), victims)
                                for u, al, uid in vs])
    status = np.zeros(n, np.int32); score = np.zeros(n, np.int32); masks = np.zeros((n, e.n_masks), e.mask_dtype)
    args = [cap._p(x) for x in (units,)] + [n] + [cap._p(x) for x in (ids, off, recs, status, score, masks)]

    def call():
        rc = e.L.egs_evict_fit(e.h, len(req), *args)
        assert rc == 0, rc
    call()                                                     # warm-up: module load, buffers
    times = []
    for _ in range(a.reps):
        t = time.perf_counter()
        call()
        times.append(time.perf_counter() - t)
    assert all(np.array_equal(x, y) for x, y in zip((status, score, masks), e.evict_fit(req, ids, victims)))

    seq = []
    equal = True
    for i in range(min(a.seq_nodes, len(ids))):
        n = int(ids[i])
        t = time.perf_counter()
        e.checkpoint_save()
        for u, al, uid in victims[i]:
            e.pod_cancel(n, u, al, uid)
        fit = int(e.filter([n], req)[0])
        _, sc = e.score([n], req)
        bst, lists = e.bind(n, req, 1 << 62) if fit else (cap.EGS_ERR_NOFIT, None)
        e.checkpoint_rollback()
        seq.append(time.perf_counter() - t)
        equal &= (fit == 0) == (status[i] == cap.EGS_ERR_NOFIT) and int(sc[0]) == int(score[i]) and bst == status[i]
        equal &= bst != 0 or lists == cap.masks_to_lists(masks[i], len(req))
    print(json.dumps(dict(
        card=card(), nodes=w.n_nodes, history_pods=a.history, pending=req, candidates=len(ids),
        victims=sum(map(len, victims)), fits=int((status != cap.EGS_ERR_NOFIT).sum()),
        evict_fit_ms_median=round(1e3 * statistics.median(times), 3), evict_fit_ms_all=[round(1e3 * x, 3) for x in times],
        sequence=dict(nodes=len(seq), ms_per_node_median=round(1e3 * statistics.median(seq), 3),
                      ms_per_node_mean=round(1e3 * statistics.mean(seq), 3), equals_evict_fit=bool(equal)),
    )))


if __name__ == "__main__":
    main()
