"""The oracle driver for candidate node sets (egs_schedule_batch_nodes): the driver rule on the C oracle pod by pod
with its own verbs, each pod filtering only the node list kube-scheduler would pass it.  A helper module for
tests/test_gpu_node_sets.py and its CPU self-test tests/test_node_sets_host.py, not a test module.

Importing this module loads neither libegs nor a GPU."""
import numpy as np

from oracle_harness import M64, pod_request


def oracle_batch_nodes(o, c_off, units, uids, node_ids):
    """node_ids[p] is the ascending node-id list of pod p: filter those nodes, score the fit ones, bind the first
    maximal.  The masks keep all 16 GPUs and, when a pod has more than 4 containers, 8 planes (EGS_MASKS_PER_POD of
    a sidecar handle)."""
    mix = o.L.egso_mix64
    P = len(c_off) - 1
    planes = 8 if any(c_off[p + 1] - c_off[p] > 4 for p in range(P)) else 4
    out = dict(node=np.full(P, -1, np.int32), status=np.zeros(P, np.int32), alloc_mask=np.zeros((P, planes), np.uint16),
               fit_count=np.zeros(P, np.int32), fit_digest=np.zeros(P, np.uint64), score_digest=np.zeros(P, np.uint64))
    for p in range(P):
        req = pod_request(units, c_off, p)
        cand = np.ascontiguousarray(node_ids[p], np.int32)
        ids = cand[o.filter(cand, req).astype(bool)] if len(cand) else cand
        out["fit_count"][p] = len(ids)
        if len(ids) == 0:
            out["status"][p] = 1
            continue
        st, sc = o.score(ids, req)
        assert st == 0
        fd = sd = 0
        for i, s in zip(ids, sc):
            fd = (fd + mix(2 * int(i) + 1)) & M64
            sd = (sd + mix(2 * int(i) + 2) * (2 * int(s) + 1)) & M64
        out["fit_digest"][p], out["score_digest"][p] = fd, sd
        w = int(ids[int(np.argmax(sc))])
        st, alloc = o.bind(w, req, int(uids[p]))
        out["node"][p], out["status"][p] = w, st
        if st == 0:
            for c, a in enumerate(alloc):
                out["alloc_mask"][p, c] = sum(1 << g for g in a)
    return out
