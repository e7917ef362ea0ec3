"""The rounds engine (EGS_MODE_ROUNDS) at every resolver geometry, against the C oracle.

A batch runs under one of four geometries, chosen by its number of distinct request shapes (`mw_dispatch` and
`batch_rounds` in csrc/egs_rounds_impl.cuh):

    distinct shapes   resolver                                          tracked slots / list depth
    1-16              MwInst16, pre-install + payload prefetch          512 / 128
    17-32             MwInst32, pre-install + payload prefetch          256 / 64
    33-96             MwInst96                                          128 / 32
    > 96              MwInst96, the host forms the set of every round   128 / 32

Every case here checks, against oracle_c.OracleC run on the same cluster and pods: the six per-pod outputs, every
node's rows, and the option cache (presence, score, per-container GPU masks) of the batch's shapes; that RESCAN gives
the same outputs; and, from egs_rounds_stats and the evaluate-launch counter, that the batch took the path it is
meant to take.  A wrong option-state conversion can leave one batch's outputs right and the next batch wrong, so the
caches are compared, and a second test carries one handle through many batches and single-pod verbs.
"""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle_c as oc

pytestmark = pytest.mark.gpu

FIELDS = ["node", "status", "alloc_mask", "fit_count", "fit_digest", "score_digest"]
STOPS = ["stop_limit", "stop_shape", "stop_tracked_full", "stop_list_dry"]
RSMAX = 96                                   # shapes per round set
FRAC_CORES = (0, 5, 10, 20, 25, 40, 50)
MEMS = (16384, 24576, 40960, 81920)          # MiB per GPU


def _egs():
    import egs_b200
    return egs_b200


# ------------------------------------------------------------------------------------------------ batch generator
def _frac(rng):
    return (int(rng.choice(FRAC_CORES)), 256 * int(rng.integers(1, 161)), 0)


def _unit(rng):
    k = rng.integers(0, 8)
    if k == 0:
        return (-1, -1, 0)                   # container without a GPU request: adds 1 to a GPU, round not monotone
    if k == 1:
        return (0, 0, int(rng.integers(1, 3)))   # whole GPUs
    return _frac(rng)


def _shape(rng, kind):
    if kind == "frac":                       # single fractional container: fast path, trade_lane_key
        return (_frac(rng),)
    if kind == "multi":                      # 2-4 containers: general_pod
        return tuple(_unit(rng) for _ in range(int(rng.integers(2, 5))))
    if kind == "sentinel":
        return tuple(_frac(rng) for _ in range(int(rng.integers(0, 3)))) + ((-1, -1, 0),)
    return ((0, 0, int(rng.integers(1, 3))),) + tuple(_frac(rng) for _ in range(int(rng.integers(0, 2))))   # whole


def _shapes(rng, n, kinds):
    """n distinct shapes.  kinds: "single" (fractional single-container only), "mixed" (all four kinds) or "multi"
    (2-4 containers only)."""
    pick = {"single": ["frac"], "mixed": ["frac", "frac", "multi", "sentinel", "whole"], "multi": ["multi"]}[kinds]
    out, seen = [], set()
    while len(out) < n:
        sh = _shape(rng, pick[int(rng.integers(0, len(pick)))])
        if sh not in seen:
            seen.add(sh); out.append(sh)
    return out


def _nodes(rng, n_nodes):
    """Heterogeneous nodes (G in 1, 2, 4, 8; up to 81920 MiB per GPU); about half start partly used."""
    nodes = []
    for _ in range(n_nodes):
        g, m = int(rng.choice([1, 2, 4, 8])), int(rng.choice(MEMS))
        rows = None
        if rng.integers(0, 2):
            rows = ([int(rng.choice([100, 100, 60, 30, 0])) for _ in range(g)], [int(rng.integers(0, m + 1)) for _ in range(g)])
        nodes.append((g, m, rows))
    return nodes


def _pods(rng, shapes, n_pods, arrival):
    """Pod -> shape index.  "front": every shape in the first pods, then uniform picks.  "trickle": six phases; phase
    i picks among a window of 64 shapes that moves on by 40 shapes a phase (cyclically), each shape's first pod at
    the start of its first phase.  Above 96 shapes a round that runs into the next phase meets more than 96 distinct
    shapes, so the host-formed sets hold part of the batch's shapes and change from round to round."""
    n = len(shapes)
    if arrival == "front":
        rest = rng.integers(0, n, max(0, n_pods - n))
        return np.concatenate([np.arange(min(n, n_pods)), rest]).astype(np.int64)
    assert arrival == "trickle"
    w, span, seen, out = min(64, n), n_pods // 6, set(), []
    for i in range(6):
        window = [(40 * i + t) % n for t in range(w)]
        new = [s for s in window if s not in seen]
        seen.update(new)
        m = n_pods - len(out) if i == 5 else span
        out += new + [window[int(j)] for j in rng.integers(0, w, m - len(new))]
    assert len(seen) == n and len(out) == n_pods
    return np.array(out, np.int64)


class Batch:
    def __init__(self, policy, nodes, shapes, pick):
        self.policy, self.nodes, self.shapes = policy, nodes, shapes
        self.n_nodes, self.n_pods = len(nodes), len(pick)
        c_off, units = [0], []
        for s in pick:
            units.extend(shapes[int(s)])
            c_off.append(len(units))
        self.c_off = np.array(c_off, np.int32)
        self.units = np.array(units, np.int32).reshape(-1, 3)


def _batch(seed, n_nodes, n_shapes, n_pods, policy, kinds, arrival):
    rng = np.random.default_rng(seed)
    nodes = _nodes(rng, n_nodes)
    shapes = _shapes(rng, n_shapes, kinds)
    return Batch(policy, nodes, shapes, _pods(rng, shapes, n_pods, arrival))


def _antichain_batch(seed, n_shapes, per_shape, n_pods, policy):
    """Shape k = (core k, mem 81920 - 512 k) on one-GPU nodes, per_shape nodes of each type k whose only GPU has
    exactly (k, 81920 - 512 k) free: type k fits shape k and no other, and one pod fills it.  Four more node
    types are full nodes that fit nothing, so that no k_select CTA (512 nodes) sees 32 nodes of one shape and
    the merged lists are exact: every shape's list holds all its nodes (no list can run dry) and every pod wins on a
    node not yet tracked, so the tracked table fills however large it is."""
    rng = np.random.default_rng(seed)
    assert n_shapes <= RSMAX
    shapes = [((k, 81920 - 512 * k, 0),) for k in range(n_shapes)]
    types = [([k], [81920 - 512 * k]) for k in range(n_shapes)] + [([0], [0])] * 4
    nodes = [(1, 81920, rows) for _ in range(per_shape) for rows in types]
    return Batch(policy, nodes, shapes, _pods(rng, shapes, n_pods, "front"))


def _distinct_shapes(b):
    """Distinct shapes of the batch as the library sees them (workloads.shapes_of's counting)."""
    seen, out = set(), []
    for p in range(b.n_pods):
        u = tuple(tuple(int(x) for x in b.units[k]) for k in range(int(b.c_off[p]), int(b.c_off[p + 1])))
        if u not in seen:
            seen.add(u); out.append(u)
    return out


def _load(e, nodes):
    for n, (g, m, rows) in enumerate(nodes):
        assert e.node_set_allocatable(n, 100 * g, m * g) == 0
        if rows is not None:
            assert e.state_load(n, rows[0], rows[1]) == 0


def _gpu(b, world=1, rank=0):
    e = _egs().Egs(b.policy, b.n_nodes)
    if world > 1:
        e.shard_set(rank, world)
    _load(e, b.nodes)
    return e


def _oracle(policy, nodes):
    o = oc.OracleC(policy)
    for n, (g, m, rows) in enumerate(nodes):
        assert o.add_node(100 * g, m * g) == n
        if rows is not None:
            o.set_rows(n, rows[0], rows[1])
    return o


# ------------------------------------------------------------------------------------------------ comparison
def _oracle_cache(o, sh, nodes):
    """The oracle's option cache of shape `sh` on `nodes`: (present, score, masks [n, 4])."""
    L, units, nc = o.L, oc._units(sh), len(sh)
    off, idx, sc = np.zeros(nc + 1, np.int32), np.zeros(16 * nc + 1, np.int32), C.c_int64(0)
    offp, idxp = off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p)
    present = np.zeros(len(nodes), bool)
    score = np.zeros(len(nodes), np.int64)
    masks = np.zeros((len(nodes), 4), np.uint8)
    for i, n in enumerate(nodes):
        if L.egso_peek(o.h, int(n), nc, units, C.byref(sc), offp, idxp):
            present[i], score[i] = True, sc.value
            for c in range(nc):
                masks[i, c] = sum(1 << int(g) for g in idx[off[c]:off[c + 1]])
    return present, score, masks


def _oracle_fits(o, sh, nodes):
    """Whether Trade of shape `sh` succeeds on the oracle's current rows of each of `nodes` (no side effects)."""
    L, units, nc = o.L, oc._units(sh), len(sh)
    off, idx, sc = np.zeros(nc + 1, np.int32), np.zeros(16 * nc + 1, np.int32), C.c_int64(0)
    offp, idxp = off.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p)
    return np.array([L.egso_trade(o.h, int(n), nc, units, offp, idxp, C.byref(sc)) == 0 for n in nodes], bool)


def _compare_caches(e, o, shapes, nodes, unfit_check):
    """Option cache of every shape on `nodes`: presence, score and masks equal the oracle's.  With unfit_check, a
    node the library marks "known not to fit" (option_dump state 2) must not fit in the oracle either."""
    nodes = np.asarray(sorted(nodes), np.int64)
    for sh in shapes:
        st, sc, am = e.option_dump(list(sh))
        st, sc, am = st[nodes], sc[nodes], am[nodes]
        present, score, masks = _oracle_cache(o, sh, nodes)
        bad = np.nonzero(present != (st == 1))[0]
        assert bad.size == 0, f"shape {sh}: cache presence differs on nodes {nodes[bad[:5]].tolist()} " \
                              f"(library state {st[bad[:5]].tolist()})"
        assert np.array_equal(score[present], sc[present].astype(np.int64)), f"shape {sh}: cached score differs"
        assert np.array_equal(masks[present], am[present]), f"shape {sh}: cached GPU masks differ"
        if unfit_check:
            unfit = nodes[st == 2]
            fits = _oracle_fits(o, sh, unfit)
            assert not fits.any(), f"shape {sh}: nodes {unfit[fits][:5].tolist()} marked unfit but fit"


def _compare_rows(e, o, n_nodes):
    core, mem, gc, _ = e.state_dump()
    for n in range(n_nodes):
        rows = o.rows(n)
        assert [(int(core[n, g]), int(mem[n, g])) for g in range(int(gc[n]))] == rows, f"rows of node {n}"


def _compare_outputs(ref, got, what):
    for f in FIELDS:
        bad = np.nonzero(ref[f] != got[f])[0]
        assert bad.size == 0, f"{what}: {f} differs first at pod {bad[:3].tolist()}"


def _delta(s1, s0):
    return {k: s1[k] - s0[k] for k in s1}


def _check_paths(d, n_shapes, n_pods):
    """egs_rounds_stats delta of one batch: every round has exactly one stop reason, every pod was resolved, and
    "shape outside the round set" occurs exactly when the host forms the sets."""
    assert sum(d[k] for k in STOPS) == d["rounds"], d
    assert d["pods"] == n_pods, d
    if n_shapes > RSMAX:
        assert d["stop_shape"] > 0, d
    else:
        assert d["stop_shape"] == 0, d


def _run_case(b, n_shapes, cache_sample=4000, threads=4):
    """ROUNDS on a fresh handle and RESCAN on another against the oracle; returns the rounds_stats delta."""
    eg = _egs()
    cap = eg.capi
    shapes = _distinct_shapes(b)
    assert len(shapes) == n_shapes
    o = _oracle(b.policy, b.nodes)
    ref = o.schedule_batch(b.c_off, b.units.astype(np.int64), threads=threads)

    e = _gpu(b)
    s0, ev0 = e.rounds_stats(), e.profile_get(cap.EGS_K_EVALUATE)[0]
    got = e.schedule_batch(b.c_off, b.units, mode=cap.EGS_MODE_ROUNDS)
    d = _delta(e.rounds_stats(), s0)
    # fresh handle: every shape is cold; one full-evaluate launch each, at most one round set's worth
    assert e.profile_get(cap.EGS_K_EVALUATE)[0] - ev0 == min(n_shapes, RSMAX)
    _compare_outputs(ref, got, "rounds")
    _check_paths(d, n_shapes, b.n_pods)
    _compare_rows(e, o, b.n_nodes)
    nodes = set(range(b.n_nodes))
    if b.n_nodes > cache_sample:
        rng = np.random.default_rng(b.n_nodes + n_shapes)
        nodes = set(int(x) for x in rng.choice(b.n_nodes, cache_sample, replace=False)) | set(int(x) for x in ref["node"] if x >= 0)
    _compare_caches(e, o, shapes, nodes, unfit_check=b.n_nodes <= 1024)
    e.close()

    r = _gpu(b)
    _compare_outputs(ref, r.schedule_batch(b.c_off, b.units, mode=cap.EGS_MODE_RESCAN), "rescan")
    r.close()
    return d, ref


# ------------------------------------------------------------------------------------------------ shape-count matrix
# Two sizes per (shape count, policy, mix):
#   pressure: 53 nodes, far more pods than fit -- NOFIT and TRANSACT outputs, unfit options, tracked tables that
#             fill with the few nodes there are; every shape arrives in the first pods.
#   wide:     2999 nodes, 6000 pods -- long lists, lists that run dry (spread) and tracked tables that fill (many
#             shapes, each winning on nodes of its own); shapes trickle in, so above 96 shapes the host-formed sets
#             change from round to round.
SIZES = {"pressure": (53, 2500, "front"), "wide": (2999, 6000, "trickle")}
INSTANCES = {"inst16": (1, 16), "inst32": (17, 32), "inst96": (33, 96), "host_formed": (97, 200)}


@pytest.mark.parametrize("inst", list(INSTANCES))
def test_round_set_matrix(inst):
    """Both shape counts of one resolver geometry (its bounds: 1/16, 17/32, 33/96, 97/200), crossed with policy
    {binpack, spread}, mix {single-container only, mixed} and the two sizes.  Over the whole set, rounds must end on
    a full tracked table and on a dry candidate list at least once each."""
    total = dict.fromkeys(["rounds", "pods", "tracked"] + STOPS, 0)
    n_nofit = n_transact = 0
    seed = 0

    def add(d, what):
        print(f"{inst} {what}: {d}")
        for k in total:
            total[k] += d[k]
    for n_shapes in INSTANCES[inst]:
        for policy in (0, 1):
            for kinds in ("single", "mixed"):
                for size, (n_nodes, n_pods, arrival) in SIZES.items():
                    seed += 1
                    b = _batch(1000 * n_shapes + seed, n_nodes, n_shapes, n_pods, policy, kinds, arrival)
                    d, ref = _run_case(b, n_shapes)
                    add(d, f"n_shapes={n_shapes} policy={policy} {kinds} {size}")
                    if size == "pressure":
                        assert (ref["status"] == 1).sum() > 0, "pressure case without NOFIT"
                        n_nofit += int((ref["status"] == 1).sum()); n_transact += int((ref["status"] == 3).sum())
    n_shapes = INSTANCES[inst][1]
    if n_shapes <= RSMAX:
        # the tracked-full case: one-pod nodes, every pod a new tracked node.  Random clusters do not fill the
        # 512-slot table of the 16-shape resolver: their shapes' lists share most nodes and run dry first.
        per_shape = max(20, 1600 // n_shapes)
        for policy in (0, 1):
            b = _antichain_batch(policy, n_shapes, per_shape, per_shape * n_shapes + 400, policy)
            d, _ = _run_case(b, n_shapes)
            add(d, f"n_shapes={n_shapes} policy={policy} one-pod nodes")
            assert d["stop_tracked_full"] > 0 and d["stop_list_dry"] == 0, d
    print(f"{inst} total: {total} nofit={n_nofit} transact={n_transact}")
    if inst == "host_formed":
        assert total["stop_shape"] > len(INSTANCES[inst]) * 8, total   # more than one per case on average
    assert total["stop_tracked_full"] > 0, total
    assert total["stop_list_dry"] > 0, total
    assert n_transact > 0


# ------------------------------------------------------------------------------------------------ state across batches
def _verbs_between(rng, e, o, shapes, n_nodes, last, uid):
    """The same single-pod verbs on both sides: filter on a node subset, bind on a fit node, AddPod of a pod another
    scheduler placed, ForgetPod of a pod the last batch placed.  Returns the next free uid."""
    for _ in range(4):
        sh = list(shapes[int(rng.integers(0, len(shapes)))])
        ids = np.sort(rng.choice(n_nodes, 300, replace=False)).astype(np.int32)
        fe, fo = e.filter(ids, sh), o.filter(ids, sh)
        assert np.array_equal(fe, fo), f"filter {sh}"
        fit = ids[fe == 1]
        if fit.size:
            node = int(fit[int(rng.integers(0, fit.size))])
            assert e.bind(node, sh, uid) == o.bind(node, sh, uid), f"bind {sh} on node {node}"
            uid += 1
    node = int(rng.integers(0, n_nodes))
    g = o.gpu_count(node)
    req, alloc = [(10, 512, 0), (-1, -1, 0)], [[int(rng.integers(0, g))], []]
    assert e.pod_apply(node, req, alloc, uid) == 0 and o.add_pod(node, req, alloc, uid) == 0
    uid += 1
    placed = [(p, int(last["node"][p])) for p in range(len(last["node"])) if last["status"][p] == 0]
    for p, node in [placed[int(i)] for i in rng.choice(len(placed), min(3, len(placed)), replace=False)]:
        sh = last["shapes"][p]
        alloc = [[gi for gi in range(8) if int(last["alloc_mask"][p][c]) >> gi & 1] for c in range(len(sh))]
        assert e.pod_cancel(node, list(sh), alloc, int(last["uids"][p])) == 0
        o.forget_pod(node, list(sh), alloc, int(last["uids"][p]))
    return uid


def _run_batches(e, o, rng, nodes, policy, plan, n_pods, every_batch=True):
    """One handle, one oracle: batch k brings plan[k] = (old, new) shapes -- `old` already interned, `new` not.
    every_batch: after every batch, the caches of all interned shapes on all nodes; else only after the last batch,
    its own shapes on all nodes and all interned shapes on 64 sampled nodes.  Returns the interned shapes."""
    interned, pool = [], _shapes(rng, sum(n for _, n in plan), "mixed")
    uid = 1 << 40
    last = None
    for k, (n_old, n_new) in enumerate(plan):
        if last is not None:
            uid = _verbs_between(rng, e, o, interned, len(nodes), last, uid)
        old = [interned[int(i)] for i in rng.choice(len(interned), min(n_old, len(interned)), replace=False)] if interned else []
        new = pool[:n_new]; pool = pool[n_new:]
        shapes = old + new
        pick = _pods(rng, shapes, n_pods, "trickle" if k % 2 and len(shapes) <= RSMAX else "front")
        b = Batch(policy, nodes, shapes, pick)
        uids = np.arange(uid, uid + n_pods, dtype=np.uint64); uid += n_pods
        ref = o.schedule_batch(b.c_off, b.units.astype(np.int64), uids=uids, threads=4)
        s0 = e.rounds_stats()
        got = e.schedule_batch(b.c_off, b.units, uids=uids, mode=2)
        _compare_outputs(ref, got, f"batch {k} ({len(shapes)} shapes)")
        _check_paths(_delta(e.rounds_stats(), s0), len(_distinct_shapes(b)), n_pods)
        interned += new
        _compare_rows(e, o, len(nodes))
        if every_batch:
            _compare_caches(e, o, interned, range(len(nodes)), unfit_check=True)
        elif k == len(plan) - 1:
            _compare_caches(e, o, shapes, range(len(nodes)), unfit_check=True)
            _compare_caches(e, o, interned, rng.choice(len(nodes), 64, replace=False), unfit_check=True)
        last = dict(ref, uids=uids, shapes=[shapes[int(s)] for s in pick])
    return interned


def test_state_across_batches():
    """One handle through seven batches, each bringing 45 new shapes next to older ones (45 to 115 shapes a batch,
    so both the one-set and the host-formed path run), with filter / bind / AddPod / ForgetPod in between.  The
    option tables grow 16 -> 512 slots while older shapes hold stale cached options; after every batch the cache of
    EVERY shape interned so far must equal the oracle's, not only the outputs."""
    eg = _egs()
    rng = np.random.default_rng(77)
    nodes = _nodes(rng, 1000)
    for policy in (0, 1):
        e, o = eg.Egs(policy, len(nodes)), _oracle(policy, nodes)
        _load(e, nodes)
        plan = [(0, 45), (20, 45), (40, 45), (60, 45), (30, 45), (70, 45), (50, 45)]
        interned = _run_batches(e, o, rng, nodes, policy, plan, 1500)
        assert len(interned) == 315
        e.close()


def test_more_than_4096_shapes():
    """On 1000 nodes (about 9 B per node per shape slot, so some 40 MB of option tables), five batches intern
    4250 shapes; past 4096 the per-shape observation flags are reallocated.  The last batch must still match the
    oracle: outputs, rows and the caches of every shape."""
    eg = _egs()
    rng = np.random.default_rng(4097)
    nodes = _nodes(rng, 1000)
    e, o = eg.Egs(1, len(nodes)), _oracle(1, nodes)
    _load(e, nodes)
    plan = [(0, 850), (40, 850), (40, 850), (40, 850), (40, 850)]
    interned = _run_batches(e, o, rng, nodes, 1, plan, 1200, every_batch=False)
    assert len(interned) == 4250
    e.close()


# ------------------------------------------------------------------------------------------------ sharded parity
@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_round_sets_equal_unsharded(world):
    """In-process shard group (egs_comm_init_local, one thread per rank) with 24 multi-container shapes, 96 shapes
    and 200 shapes (host-formed sets).  Every rank's outputs equal the unsharded run and every shard's rows equal
    the unsharded rows.  At world 8 the 96-shape resolver keeps rke = 4 list entries per (shape, shard) in shared
    memory -- MwSmem<96, 128> takes 196 264 B of the 232 448 B, the lists 96 x 8 x 8 B per entry -- the floor
    below which batch_rounds refuses; it must schedule there."""
    eg = _egs()
    cap = eg.capi
    for n_shapes, kinds, arrival in [(24, "multi", "front"), (96, "mixed", "front"), (200, "mixed", "trickle")]:
        b = _batch(world * 1000 + n_shapes, 2500, n_shapes, 4000, 1, kinds, arrival)
        assert len(_distinct_shapes(b)) == n_shapes
        e0 = _gpu(b)
        ref = e0.schedule_batch(b.c_off, b.units, mode=cap.EGS_MODE_ROUNDS)
        ref_core, ref_mem, _, _ = e0.state_dump()
        e0.close()
        hs = [_gpu(b, world, r) for r in range(world)]
        cap.comm_init_local(hs)
        outs, errs = [None] * world, []

        def run(r):
            try:
                outs[r] = hs[r].schedule_batch(b.c_off, b.units, mode=cap.EGS_MODE_ROUNDS)
            except Exception as ex:   # pragma: no cover
                errs.append(repr(ex))
        th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
        for t in th:
            t.start()
        for t in th:
            t.join(timeout=600)
        assert not errs, errs
        for r in range(world):
            _compare_outputs(ref, outs[r], f"{n_shapes} shapes, world {world}, rank {r}")
            lo, hi = cap.shard_range(b.n_nodes, r, world)
            core, mem, _, _ = hs[r].state_dump(lo, hi - lo)
            assert np.array_equal(core, ref_core[lo:hi]) and np.array_equal(mem, ref_mem[lo:hi]), f"rows of shard {r}"
        for e in hs:
            e.close()
