"""Clusters with a history for the headroom tests, and the check that a headroom answer equals a dry run.

A history is a batch of mixed pods, which caches options and "does not fit" marks for every shape of the mix, followed
by AddPod records that change rows under those cached options, so that some of them are stale.  Nodes start fresh,
partly used, or with GPUs above their totals.  The same cluster and history run on a library handle
(schedule_batch_mut) and on the oracle (oracle_harness.oracle_batch).

Importing this module loads neither libegs nor a GPU."""
import numpy as np

SENT = (-1, -1, 0)
NOFIT, TRANSACT = 1, 3


def nodes(rng, n, gpus=(1, 2, 4, 8), mems=(16, 40)):
    """n nodes [(gpu_count, mem_total per GPU, (core row, mem row) or None)].  A third start fresh; the others have
    GPUs free, partly used, empty, or above their totals (a row loaded over them)."""
    out = []
    for _ in range(n):
        g, mt = int(rng.choice(gpus)), int(rng.choice(mems))
        if rng.integers(0, 3) == 0:
            out.append((g, mt, None))
            continue
        core, mem = [], []
        for _ in range(g):
            k = rng.integers(0, 4)
            if k == 0:
                c, m = 100, mt
            elif k == 1:
                c, m = int(rng.choice([0, 10, 35, 60, 90])), int(rng.integers(0, mt + 1))
            elif k == 2:
                c, m = int(rng.integers(100, 140)), mt + int(rng.integers(0, mt // 4 + 3))
            else:
                c, m = 0, 0
            core.append(c); mem.append(m)
        out.append((g, mt, (core, mem)))
    return out


def pods(shapes, pick):
    """c_off, units of one pod per entry of `pick` (indices into shapes)."""
    units = np.array([u for p in pick for u in shapes[p]], np.int32).reshape(-1, 3)
    c_off = np.concatenate([[0], np.cumsum([len(shapes[p]) for p in pick])]).astype(np.int32)
    return c_off, units


def identical(shape, k):
    """k pods of one shape."""
    return pods([shape], [0] * k)


def history(rng, cl_nodes, shapes, n_pods, n_add, uid0=1):
    """A batch of n_pods pods drawn from `shapes`, then n_add AddPod records on random set nodes after the last pod.
    Each record puts one fractional container on one GPU of the node: the node's rows change and its cached options
    stay, so some become stale.  Returns (c_off, units, uids, mut_at, records) for schedule_batch_mut / oracle_batch."""
    c_off, units = pods(shapes, rng.integers(0, len(shapes), n_pods))
    uids = np.arange(uid0, uid0 + n_pods, dtype=np.uint64)
    live = [n for n, nd in enumerate(cl_nodes) if nd is not None]
    records = []
    for k in range(n_add):
        n = int(rng.choice(live))
        g, mt, _ = cl_nodes[n]
        u = (int(rng.choice([5, 10, 25])), max(1, mt // int(rng.choice([4, 8, 16]))), 0)
        records.append((0, n, [u], [[int(rng.integers(0, g))]], uid0 + n_pods + k))
    return c_off, units, uids, [n_pods] * n_add, records


def check_dry_run(count, failed, out, node0=0, what=""):
    """The headroom answer (count, failed over nodes [node0, node0 + len(count))) equals the dry run `out` of K
    identical pods over every node: per node, the EGS_OK pods won there and the EGS_ERR_TRANSACT pods there; every pod
    after the last bind is EGS_ERR_NOFIT."""
    st, nd = out["status"], out["node"]
    n_bind = int(count.sum() + failed.sum())
    assert len(st) > n_bind, f"{what}: the dry run is not longer than the answer"
    assert (st[:n_bind] != NOFIT).all() and (st[n_bind:] == NOFIT).all(), \
        f"{what}: {int((st != NOFIT).sum())} binds in the dry run, {n_bind} in the answer"
    hi = node0 + len(count)
    ok = np.bincount(nd[st == 0], minlength=hi)[node0:hi]
    bad = np.nonzero(ok != count)[0]
    assert bad.size == 0, f"{what}: node {node0 + int(bad[0])} takes {ok[bad[0]]} pods in the dry run, {count[bad[0]]} counted"
    tf = np.bincount(nd[st == TRANSACT], minlength=hi)[node0:hi]
    bad = np.nonzero(tf != failed)[0]
    assert bad.size == 0, f"{what}: node {node0 + int(bad[0])} fails {tf[bad[0]]} Transacts, {failed[bad[0]]} counted"


def summary_of(count, failed, capped=None):
    """The four summary values of one shape."""
    return [int(count.sum()), int((count > 0).sum()), int(failed.sum()), 0 if capped is None else int(np.sum(capped))]
