"""One cluster on a library handle and on the C oracle, and the comparisons the GPU tests make between them: the six
per-pod outputs, node rows, option caches, an in-process shard group against the unsharded run, and the one pod-by-pod
oracle driver, whose masks keep all 16 GPUs.

Importing this module loads neither libegs nor a GPU: `egs()` imports the package on first use."""
import threading

import numpy as np

import oracle_c as oc

FIELDS = ["node", "status", "alloc_mask", "fit_count", "fit_digest", "score_digest"]
M64 = (1 << 64) - 1


def egs():
    import egs_b200
    return egs_b200


class Cluster:
    """nodes: [(gpu_count, mem_total per GPU, (core row, mem row) or None)].  The same cluster on a library handle
    (rows through egs_state_load, or egs_state_load_bulk for a workload) and on the oracle.  A cluster of a workload
    (anything with policy, n_nodes, gpus, mem_total and core / mem [n_nodes, gpus]) is loaded in bulk on both sides,
    and its node list is only built when asked for.  c_max > 4 makes the handle a sidecar handle.  A None node is an id
    never set on the handle; the oracle, whose ids are dense, holds a 1-GPU placeholder there that a test never lists."""

    def __init__(self, policy, nodes, g_max=8, c_max=4):
        self.policy, self._nodes, self.g_max, self.c_max = policy, nodes, g_max, c_max
        self.workload = None

    @classmethod
    def of_workload(cls, w, g_max=8):
        cl = cls(w.policy, None, g_max)
        cl.workload = w
        return cl

    @property
    def nodes(self):
        if self._nodes is None:
            w = self.workload
            self._nodes = [(w.gpus, w.mem_total, (w.core[n], w.mem[n])) for n in range(w.n_nodes)]
        return self._nodes

    @property
    def n_nodes(self):
        return self.workload.n_nodes if self.workload is not None else len(self._nodes)

    def handle(self, world=1, rank=0):
        e = egs().Egs(self.policy, self.n_nodes, self.g_max, c_max=self.c_max)
        if world > 1:
            e.shard_set(rank, world)
        w = self.workload
        if w is not None:
            e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
            return e
        for n, nd in enumerate(self.nodes):
            if nd is None:
                continue
            g, mt, rows = nd
            assert e.node_set_allocatable(n, 100 * g, mt * g) == 0
            if rows is not None:
                assert e.state_load(n, rows[0], rows[1]) == 0
        return e

    def oracle(self):
        o = oc.OracleC(self.policy)
        w = self.workload
        if w is not None:
            assert o.add_nodes(w.gpus, w.mem_total * w.gpus, w.core, w.mem) == 0
            return o
        for n, nd in enumerate(self.nodes):
            g, mt, rows = nd or (1, 1, None)
            assert o.add_node(100 * g, mt * g) == n
            if rows is not None:
                o.set_rows(n, rows[0], rows[1])
        return o


def compare_outputs(ref, got, what):
    for f in FIELDS:
        bad = np.nonzero(ref[f] != got[f])[0]
        assert bad.size == 0, f"{what}: {f} differs first at pod {bad[:3].tolist()}"


def compare_rows(e, o, nodes):
    """Rows of `nodes`: the library's first gpu_count cells are the oracle's rows and every cell past them is PAD."""
    cap = egs().capi
    core, mem, gc, _ = e.state_dump()
    W = core.shape[1]
    assert W == cap.row_width(e.g_max)
    nodes = np.unique(np.fromiter(nodes, np.int64))
    core, mem, gc = core[nodes], mem[nodes], gc[nodes]
    ocore, omem, ogc = o.rows_many(nodes, W)
    bad = np.nonzero(gc != ogc)[0]
    assert bad.size == 0, f"rows of node {int(nodes[bad[0]])}: {gc[bad[0]]} GPUs, the oracle has {ogc[bad[0]]}"
    live = np.arange(W)[None, :] < ogc[:, None]
    bad = np.nonzero((live & ((core != ocore) | (mem != omem))).any(1))[0]
    assert bad.size == 0, f"rows of node {int(nodes[bad[0]])}"
    bad = np.nonzero((~live & ((core != cap.EGS_PAD) | (mem != cap.EGS_PAD))).any(1))[0]
    assert bad.size == 0, f"PAD cells of node {int(nodes[bad[0]])}"


def compare_caches(e, o, shapes, nodes, unfit_check):
    """Option cache of every shape on `nodes`: presence, score and masks equal the oracle's, at the mask width and
    plane count of the handle's option_dump (u8, or u16 on a wide handle; 4 planes, or 8 on a sidecar handle).  With
    unfit_check, a node the library marks "known not to fit" (option_dump state 2) must not fit in the oracle either."""
    nodes = np.asarray(sorted(nodes), np.int64)
    for sh in shapes:
        st, sc, am = e.option_dump(list(sh))
        assert am.dtype == egs().capi.mask_dtype(e.g_max), f"shape {sh}: mask dtype {am.dtype}"
        assert am.shape[1] == e.n_masks, f"shape {sh}: {am.shape[1]} mask planes"
        st, sc, am = st[nodes], sc[nodes], am[nodes]
        present, score, masks = o.peek_many(nodes, sh, e.n_masks)
        bad = np.nonzero(present != (st == 1))[0]
        assert bad.size == 0, f"shape {sh}: cache presence differs on nodes {nodes[bad[:5]].tolist()} " \
                              f"(library state {st[bad[:5]].tolist()})"
        assert np.array_equal(score[present], sc[present].astype(np.int64)), f"shape {sh}: cached score differs"
        assert np.array_equal(masks[present], am[present]), f"shape {sh}: cached GPU masks differ"
        if unfit_check:
            unfit = nodes[st == 2]
            fits = o.trade_fits(unfit, sh)
            assert not fits.any(), f"shape {sh}: nodes {unfit[fits][:5].tolist()} marked unfit but fit"


def conservation(w, out, e):
    """Size-independent property: final rows == initial rows - sum of successful binds."""
    core = w.core.astype(np.int64).copy()
    mem = w.mem.astype(np.int64).copy()
    ok = out["status"] == 0
    assert ((out["node"] >= 0) == (out["status"] != 1)).all()
    for c in range(4):
        has = ok & (np.diff(w.c_off) > c)
        pods = np.nonzero(has)[0]
        m = out["alloc_mask"][pods, c]
        assert (np.bitwise_count(m) == 1).all()
        g = np.log2(m.astype(np.float64)).astype(np.int64)
        u = w.units[w.c_off[pods] + c]
        np.subtract.at(core, (out["node"][pods], g), u[:, 0])
        np.subtract.at(mem, (out["node"][pods], g), u[:, 1])
    dc, dm, _, _ = e.state_dump()
    assert np.array_equal(dc[:, :w.gpus], core) and np.array_equal(dm[:, :w.gpus], mem)
    assert (core >= 0).all() and (mem >= 0).all()


def late_window(cfg, policy, K, W, n_nodes=None, threads=4, sample=4000):
    """The GPU engine schedules the first K pods of config `cfg` (at `n_nodes`, default its named size); rows and
    every option cache are dumped through the ABI and loaded into a FRESH oracle (egso_cache_load); both then schedule
    pods [K, K+W) and must agree on all six outputs, the final rows and the final caches.  This puts the oracle into
    the late, full-cluster regime (stale options, bind failures, unfit nodes) that a prefix from an empty cluster
    never reaches.  Returns the window's outputs and the handle."""
    eg = egs()
    full = eg.workloads.config(cfg, n_nodes=n_nodes, n_pods=K + W, policy=policy)
    e = Cluster.of_workload(full).handle()
    pre = full.prefix(K)
    e.schedule_batch(pre.c_off, pre.units, mode=2)
    core, mem, _, _ = e.state_dump()
    o = oc.OracleC(full.policy)
    assert o.add_nodes(full.gpus, full.mem_total * full.gpus, core[:, :full.gpus], mem[:, :full.gpus]) == 0
    shapes = eg.workloads.shapes_of(full)
    n_cached = 0
    for sh in shapes:
        st, sc, am = e.option_dump(list(sh))
        assert o.cache_load(list(sh), st == 1, sc, am) == 0
        n_cached += int((st == 1).sum())
    assert n_cached > 0
    win = eg.workloads.window(full, K, W)
    ref = o.schedule_batch(win.c_off, win.units64(), threads=threads)
    compare_outputs(ref, e.schedule_batch(win.c_off, win.units, mode=2), f"cfg{cfg} K={K}")
    rng = np.random.default_rng(K)
    nodes = set(int(x) for x in rng.integers(0, full.n_nodes, sample)) | set(int(x) for x in ref["node"] if x >= 0)
    compare_rows(e, o, nodes)
    compare_caches(e, o, shapes, nodes, unfit_check=True)
    return ref, e


# ------------------------------------------------------------------------------------------------ shard groups
def run_sharded(handle, world, c_off, units):
    """The batch under EGS_MODE_ROUNDS on handle() and on an in-process shard group (egs_comm_init_local, one thread
    per rank) of handle(world, rank).  Returns the unsharded outputs, the unsharded rows (core, mem) and, per rank,
    (outputs, first node of its shard, core and mem rows of its shard)."""
    cap = egs().capi
    e = handle()
    ref = e.schedule_batch(c_off, units, mode=cap.EGS_MODE_ROUNDS)
    rows = e.state_dump()[:2]
    e.close()
    hs = [handle(world, r) for r in range(world)]
    cap.comm_init_local(hs)
    outs, errs = [None] * world, []

    def run(r):
        try:
            outs[r] = hs[r].schedule_batch(c_off, units, mode=cap.EGS_MODE_ROUNDS)
        except Exception as ex:   # pragma: no cover
            errs.append(repr(ex))
    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    ranks = []
    for r, h in enumerate(hs):
        lo, hi = cap.shard_range(h.max_nodes, r, world)
        ranks.append((outs[r], lo) + h.state_dump(lo, hi - lo)[:2])
        h.close()
    return ref, rows, ranks


def compare_shards(ref, rows, ranks, what):
    """Every rank's outputs equal the unsharded run's, and every shard's rows the unsharded rows."""
    for r, (out, lo, core, mem) in enumerate(ranks):
        compare_outputs(ref, out, f"{what}, rank {r}")
        hi = lo + len(core)
        assert np.array_equal(core, rows[0][lo:hi]) and np.array_equal(mem, rows[1][lo:hi]), f"{what}: rows of shard {r}"


# ------------------------------------------------------------------------------------------------ oracle driver
def pod_request(units, c_off, p):
    return [tuple(int(x) for x in units[k]) for k in range(int(c_off[p]), int(c_off[p + 1]))]


def oracle_batch(o, c_off, units, uids, muts=(), mut_at=(), node_ids=None, planes=4):
    """The driver rule on the oracle pod by pod with its own verbs -- filter the pod's nodes, score the fit ones, bind
    the first maximal -- so the masks keep all 16 GPUs (egso_schedule_batch's hold 8), in `planes` planes (4, or 8 for
    a sidecar handle).  Records muts[j] apply right before pod mut_at[j].  node_ids[p] is the ascending node list
    kube-scheduler passes pod p (egs_schedule_batch_nodes); None: every node."""
    mix = o.L.egso_mix64
    P = len(c_off) - 1
    out = dict(node=np.full(P, -1, np.int32), status=np.zeros(P, np.int32), alloc_mask=np.zeros((P, planes), np.uint16),
               fit_count=np.zeros(P, np.int32), fit_digest=np.zeros(P, np.uint64), score_digest=np.zeros(P, np.uint64))
    j = 0
    for p in range(P):
        while j < len(mut_at) and mut_at[j] == p:
            oracle_mut(o, muts[j]); j += 1
        req = pod_request(units, c_off, p)
        if node_ids is None:
            ids = np.flatnonzero(o.filter(None, req)).astype(np.int32)
        else:
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
    while j < len(mut_at):
        oracle_mut(o, muts[j]); j += 1
    return out


def oracle_mut(o, rec):
    kind, node, req, alloc, uid = rec
    if kind == 1:
        o.forget_pod(node, req, alloc, uid)
    else:                                   # ADD, and REPLAY of a uid no podsMap holds: the same row update
        o.add_pod(node, req, alloc, uid)
