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
import numpy as np
import pytest

from oracle_harness import Cluster, compare_caches, compare_outputs, compare_rows, compare_shards, egs, run_sharded
from round_batches import RSMAX, STOPS, Batch, check_paths, distinct_shapes, pod_picks, stats_delta

pytestmark = pytest.mark.gpu

FRAC_CORES = (0, 5, 10, 20, 25, 40, 50)
MEMS = (16384, 24576, 40960, 81920)          # MiB per GPU


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


def _batch(seed, n_nodes, n_shapes, n_pods, policy, kinds, arrival):
    rng = np.random.default_rng(seed)
    nodes = _nodes(rng, n_nodes)
    shapes = _shapes(rng, n_shapes, kinds)
    return Batch(policy, nodes, shapes, pod_picks(rng, shapes, n_pods, arrival))


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
    return Batch(policy, nodes, shapes, pod_picks(rng, shapes, n_pods, "front"))


def _run_case(b, n_shapes, cache_sample=4000, threads=4):
    """ROUNDS on a fresh handle and RESCAN on another against the oracle; returns the rounds_stats delta."""
    cap = egs().capi
    shapes = distinct_shapes(b)
    assert len(shapes) == n_shapes
    o = b.cluster.oracle()
    ref = o.schedule_batch(b.c_off, b.units.astype(np.int64), threads=threads)

    e = b.cluster.handle()
    s0, ev0 = e.rounds_stats(), e.profile_get(cap.EGS_K_EVALUATE)[0]
    got = e.schedule_batch(b.c_off, b.units, mode=cap.EGS_MODE_ROUNDS)
    d = stats_delta(e.rounds_stats(), s0)
    # fresh handle: every shape is cold; one full-evaluate launch each, at most one round set's worth
    assert e.profile_get(cap.EGS_K_EVALUATE)[0] - ev0 == min(n_shapes, RSMAX)
    compare_outputs(ref, got, "rounds")
    check_paths(d, n_shapes, b.n_pods)
    compare_rows(e, o, range(b.n_nodes))
    nodes = set(range(b.n_nodes))
    if b.n_nodes > cache_sample:
        rng = np.random.default_rng(b.n_nodes + n_shapes)
        nodes = set(int(x) for x in rng.choice(b.n_nodes, cache_sample, replace=False)) | set(int(x) for x in ref["node"] if x >= 0)
    compare_caches(e, o, shapes, nodes, unfit_check=b.n_nodes <= 1024)
    e.close()

    r = b.cluster.handle()
    compare_outputs(ref, r.schedule_batch(b.c_off, b.units, mode=cap.EGS_MODE_RESCAN), "rescan")
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
        alloc = egs().capi.masks_to_lists(last["alloc_mask"][p], len(sh))
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
        pick = pod_picks(rng, shapes, n_pods, "trickle" if k % 2 and len(shapes) <= RSMAX else "front")
        b = Batch(policy, nodes, shapes, pick)
        uids = np.arange(uid, uid + n_pods, dtype=np.uint64); uid += n_pods
        ref = o.schedule_batch(b.c_off, b.units.astype(np.int64), uids=uids, threads=4)
        s0 = e.rounds_stats()
        got = e.schedule_batch(b.c_off, b.units, uids=uids, mode=2)
        compare_outputs(ref, got, f"batch {k} ({len(shapes)} shapes)")
        check_paths(stats_delta(e.rounds_stats(), s0), len(distinct_shapes(b)), n_pods)
        interned += new
        compare_rows(e, o, range(len(nodes)))
        if every_batch:
            compare_caches(e, o, interned, range(len(nodes)), unfit_check=True)
        elif k == len(plan) - 1:
            compare_caches(e, o, shapes, range(len(nodes)), unfit_check=True)
            compare_caches(e, o, interned, rng.choice(len(nodes), 64, replace=False), unfit_check=True)
        last = dict(ref, uids=uids, shapes=[shapes[int(s)] for s in pick])
    return interned


def test_state_across_batches():
    """One handle through seven batches, each bringing 45 new shapes next to older ones (45 to 115 shapes a batch,
    so both the one-set and the host-formed path run), with filter / bind / AddPod / ForgetPod in between.  The
    option tables grow 16 -> 512 slots while older shapes hold stale cached options; after every batch the cache of
    EVERY shape interned so far must equal the oracle's, not only the outputs."""
    rng = np.random.default_rng(77)
    nodes = _nodes(rng, 1000)
    for policy in (0, 1):
        cl = Cluster(policy, nodes)
        e, o = cl.handle(), cl.oracle()
        plan = [(0, 45), (20, 45), (40, 45), (60, 45), (30, 45), (70, 45), (50, 45)]
        interned = _run_batches(e, o, rng, nodes, policy, plan, 1500)
        assert len(interned) == 315
        e.close()


def test_more_than_4096_shapes():
    """On 1000 nodes (about 9 B per node per shape slot, so some 40 MB of option tables), five batches intern
    4250 shapes; past 4096 the per-shape observation flags are reallocated.  The last batch must still match the
    oracle: outputs, rows and the caches of every shape."""
    rng = np.random.default_rng(4097)
    nodes = _nodes(rng, 1000)
    cl = Cluster(1, nodes)
    e, o = cl.handle(), cl.oracle()
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
    for n_shapes, kinds, arrival in [(24, "multi", "front"), (96, "mixed", "front"), (200, "mixed", "trickle")]:
        b = _batch(world * 1000 + n_shapes, 2500, n_shapes, 4000, 1, kinds, arrival)
        assert len(distinct_shapes(b)) == n_shapes
        compare_shards(*run_sharded(b.cluster.handle, world, b.c_off, b.units), f"{n_shapes} shapes, world {world}")
