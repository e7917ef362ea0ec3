"""Every engine on GPUs ABOVE their totals and at the int32 guard, against the C oracle.

A GPU can hold more than its totals (100 core, mem_total):
  * sidecar   -- a container without a GPU request is the (-1, -1) unit, and binding it ADDS 1 to a GPU (gpu.go:36-37);
  * forget    -- AddPod records the uid before Transact runs (node.go:149-150) and Cancel is unchecked (gpu.go:177-191),
                 so ForgetPod after a failed AddPod gives back what was never taken; through egs_pod_apply /
                 egs_pod_cancel and through the mutation stream of egs_schedule_batch_mut;
  * load      -- egs_state_load takes any row up to the guard (2^20 core, 2^25 MiB), whatever mem_total is.
Such a GPU is not free for a whole-GPU container (gpu.go:193-202, equality with the totals) until a fractional bind
brings it down to exactly its totals.  So a round whose requests are all >= 0 can turn an option that did not fit into
one that fits, and the rounds engine must not keep "does not fit" across such a bind.

Every case checks, against oracle_c.OracleC on the same cluster and pods: the six per-pod outputs, every node's rows,
the option caches of the batch's shapes (a node the library marks "does not fit" must not fit in the oracle), that
RESCAN gives the same outputs, and egs_filter / egs_score of every whole-GPU shape over all nodes after the batch.
The guard case drives rows and requests to the limits of DESIGN §1 through the cold evaluate, select, the fast /
general / leaf-parallel resolver paths, RESCAN and schedule_batch_vec.
"""
import numpy as np
import pytest

from oracle_harness import Cluster, compare_caches, compare_outputs, compare_rows, compare_shards, egs, run_sharded
from round_batches import Batch, check_paths, distinct_shapes, pod_picks, stats_delta
from rounds_cases import FRAC11, OVER, SIDECAR, WHOLE1, over_totals_shapes

pytestmark = pytest.mark.gpu

MEMS = (16384, 40960, 81920)                 # MiB per GPU
MAX_CORE, MAX_MEM = 1 << 20, 1 << 25         # EGS_MAX_CORE_LOAD, EGS_MAX_MEM_PER_GPU
# Pod uids, one range per source.  Every batch passes its uids: without them the oracle numbers each batch's pods
# from 0 and the library continues one counter, so a later batch would reuse an earlier batch's uids on the oracle
# side only -- and binding a uid the node already holds changes nothing (node.go:149).
UID_RECORDS, UID_SIDECAR, UID_BATCH = 1 << 40, 1 << 41, 1 << 42


def _over_nodes(cl, o):
    """Nodes with a GPU above its totals on the oracle's rows now."""
    return {n for n, (g, mt, _) in enumerate(cl.nodes) if any(c > 100 or m > mt for c, m in o.rows(n))}


def _forget_records(rng, cl, uid0):
    """AddPod of (whole GPU g, then (a, b) on GPU g) fails at its second container with GPU g taken, and ForgetPod of
    the same uid puts GPU g back to (100 + a, mt + b).  On about three GPUs in four of a free cluster."""
    recs, uid = [], uid0
    for n, (g, mt, _) in enumerate(cl.nodes):
        for gi in range(g):
            a, b = int(rng.choice(OVER)), int(rng.choice(OVER))
            if (a or b) and rng.integers(0, 4):
                req, alloc = [(0, 0, 1), (a, b, 0)], [[gi], [gi]]
                recs += [(egs().capi.EGS_MUT_ADD, n, req, alloc, uid), (egs().capi.EGS_MUT_FORGET, n, req, alloc, uid)]
                uid += 1
    return recs


def _apply_records(e, o, recs, verbs):
    """The records on the oracle, and on the library (e not None) through egs_pod_apply / egs_pod_cancel (verbs) or
    not at all (the caller passes them to egs_schedule_batch_mut)."""
    verbs = verbs and e is not None
    for kind, n, req, alloc, uid in recs:
        if kind == egs().capi.EGS_MUT_ADD:
            assert o.add_pod(n, req, alloc, uid) == 0
            if verbs:
                assert e.pod_apply(n, req, alloc, uid) == 0
        else:
            assert o.forget_pod(n, req, alloc, uid) == 0
            if verbs:
                assert e.pod_cancel(n, req, alloc, uid) == 0


def _sidecar_binds(rng, e, o, n_nodes, uid0):
    """One to three sidecar pods, each filtered on and bound to one node, on about three nodes in four (a batch would
    pile every sidecar on the one best-scoring GPU).  e is None: the oracle alone."""
    uid = uid0
    for n in range(n_nodes):
        for _ in range(int(rng.integers(1, 4)) if rng.integers(0, 4) else 0):
            assert o.filter([n], list(SIDECAR))[0] == 1
            st_o = o.bind(n, list(SIDECAR), uid)
            assert st_o[0] == 0
            if e is not None:
                assert e.filter([n], list(SIDECAR))[0] == 1
                assert e.bind(n, list(SIDECAR), uid) == st_o, f"sidecar bind on node {n}"
            uid += 1
    return uid


def _check_whole_verbs(e, o, shapes, n_nodes):
    """egs_filter / egs_score of every whole-GPU shape over all nodes equal the oracle's."""
    ids = np.arange(n_nodes, dtype=np.int32)
    for sh in shapes:
        if not any(u[2] > 0 for u in sh):
            continue
        assert np.array_equal(e.filter(ids, list(sh)), o.filter(ids, list(sh))), f"filter {sh}"
        se, sc_e = e.score(ids, list(sh))
        so, sc_o = o.score(ids, list(sh))
        assert se == so and np.array_equal(sc_e.astype(np.int64), sc_o), f"score {sh}"


def _regime(ref, b, over):
    """Whole-GPU pods the oracle bound on a node that had a GPU above its totals when the batch began."""
    whole = [bool((b.units[b.c_off[p]:b.c_off[p + 1], 2] > 0).any()) for p in range(b.n_pods)]
    return sum(1 for p in range(b.n_pods) if whole[p] and ref["status"][p] == 0 and int(ref["node"][p]) in over)


def _run_route(cl, route, b, pre=None, threads=4):
    """One batch `b` on a cluster reached by `route`, ROUNDS then RESCAN on fresh handles, both against the oracle.
    pre(e, o) brings a handle (e is None: the oracle alone) to the batch's starting state and returns mutation
    records for egs_schedule_batch_mut (route "stream") or None.  Returns (ref outputs, ROUNDS stats delta, nodes
    above their totals at batch start)."""
    cap = egs().capi
    shapes = distinct_shapes(b)
    o = cl.oracle()
    pre(None, o)
    over = _over_nodes(cl, o)
    uids = np.arange(UID_BATCH, UID_BATCH + b.n_pods, dtype=np.uint64)
    ref = o.schedule_batch(b.c_off, b.units.astype(np.int64), uids=uids, threads=threads)
    for mode in (cap.EGS_MODE_ROUNDS, cap.EGS_MODE_RESCAN):
        e = cl.handle()
        oe = cl.oracle()
        recs_e = pre(e, oe)
        s0 = e.rounds_stats()
        if recs_e:
            got = e.schedule_batch_mut(b.c_off, b.units, np.zeros(len(recs_e), np.int32), recs_e, uids=uids, mode=mode)
        else:
            got = e.schedule_batch(b.c_off, b.units, uids=uids, mode=mode)
        compare_outputs(ref, got, f"{route} mode {mode}")
        if mode == cap.EGS_MODE_ROUNDS:
            d = stats_delta(e.rounds_stats(), s0)
            compare_rows(e, o, range(len(cl.nodes)))
            compare_caches(e, o, shapes, range(len(cl.nodes)), unfit_check=True)
            # the verbs read the option table the batch left behind (egs_filter / egs_score trust its memos);
            # `o` is the oracle after the batch, so it answers the same filter / score questions
            _check_whole_verbs(e, o, shapes, len(cl.nodes))
        e.close()
    return ref, d, over


# ------------------------------------------------------------------------------------------------ the minimal case
MIN_PODS = [WHOLE1, FRAC11, WHOLE1]          # one node, one GPU of 16 MiB at (101, 17): NOFIT, bind, bind


def _min_batch(policy, pods):
    return Batch(policy, [(1, 16, None)], list(dict.fromkeys(pods)), [list(dict.fromkeys(pods)).index(s) for s in pods])


def _min_pre(route):
    """How the only GPU gets to (101, 17)."""
    req, alloc = [(0, 0, 1), (1, 1, 0)], [[0], [0]]

    def pre(e, o):
        cap = egs().capi
        if route == "sidecar":                                    # a batch of one sidecar pod
            sb = _min_batch(0, [SIDECAR])
            uids = np.array([UID_SIDECAR], np.uint64)
            r = o.schedule_batch(sb.c_off, sb.units.astype(np.int64), uids=uids)
            if e is not None:
                compare_outputs(r, e.schedule_batch(sb.c_off, sb.units, uids=uids, mode=cap.EGS_MODE_ROUNDS), "sidecar batch")
        elif route == "load":
            o.set_rows(0, [101], [17])
            if e is not None:
                assert e.state_load(0, [101], [17]) == 0
        else:                                                     # AddPod fails at its 2nd container; ForgetPod
            recs = [(cap.EGS_MUT_ADD, 0, req, alloc, UID_RECORDS), (cap.EGS_MUT_FORGET, 0, req, alloc, UID_RECORDS)]
            _apply_records(e, o, recs, verbs=route == "verbs")
            if route == "stream":
                return recs
        assert o.rows(0) == [(101, 17)]
        return None
    return pre


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("route", ["sidecar", "load", "verbs", "stream"])
def test_minimal_whole_gpu_fits_again(route, policy):
    """The only GPU at (101, 17) of (100, 16), then [whole GPU, (1, 1), whole GPU] in one batch: NOFIT, a bind that
    brings the GPU to its totals, and a whole-GPU bind on it -- the first pod's "does not fit" must not outlive the
    second pod's bind.  One round, requests all >= 0."""
    b = _min_batch(policy, MIN_PODS)
    ref, _, over = _run_route(Cluster(policy, [(1, 16, None)]), route, b, _min_pre(route))
    assert ref["node"].tolist() == [-1, 0, 0] and ref["status"].tolist() == [1, 0, 0]
    assert over == {0}


# ------------------------------------------------------------------------------------------------ random clusters
def _over_cluster(rng, n_nodes, route):
    """Route "load": every GPU at or just above its totals, a few partly used.  Other routes: a free cluster."""
    nodes = []
    for _ in range(n_nodes):
        g, mt = int(rng.choice([1, 2, 4, 8])), int(rng.choice(MEMS))
        rows = None
        if route == "load":
            rows = ([100 + int(rng.choice(OVER)) for _ in range(g)], [mt + int(rng.choice(OVER)) for _ in range(g)])
            for gi in range(g):
                if rng.integers(0, 8) == 0:
                    rows[0][gi], rows[1][gi] = 60, mt // 2
        nodes.append((g, mt, rows))
    return nodes


def _over_case(seed, route, n_shapes, n_nodes=160, n_pods=2000):
    rng = np.random.default_rng(seed)
    policy = seed % 2
    cl = Cluster(policy, _over_cluster(rng, n_nodes, route))
    shapes = over_totals_shapes(rng, n_shapes)
    b = Batch(policy, cl.nodes, shapes, pod_picks(rng, shapes, n_pods, "trickle" if n_shapes > 96 else "front"))
    recs = _forget_records(rng, cl, UID_RECORDS) if route in ("verbs", "stream") else []
    side_seed = seed + 1

    def pre(e, o):
        if route == "sidecar":
            _sidecar_binds(np.random.default_rng(side_seed), e, o, n_nodes, UID_SIDECAR)
        elif route in ("verbs", "stream"):
            _apply_records(e, o, recs, verbs=route == "verbs")
            return recs if route == "stream" else None
        return None
    return cl, b, pre


GEOMETRIES = {"inst16": 12, "inst96": 64, "host_formed": 130}


@pytest.mark.parametrize("inst", list(GEOMETRIES))
@pytest.mark.parametrize("route", ["sidecar", "load", "verbs", "stream"])
def test_random_clusters_above_totals(route, inst):
    """160 nodes of 1-8 GPUs brought above their totals by `route`, 2000 pods of `GEOMETRIES[inst]` shapes (the
    pre-install resolver, the 96-shape one, host-formed sets).  Whole-GPU pods must win on nodes that began the batch
    above their totals, or the case did not reach the regime it is here for."""
    n_shapes = GEOMETRIES[inst]
    cl, b, pre = _over_case(100 * n_shapes + len(route), route, n_shapes)
    ref, d, over = _run_route(cl, route, b, pre)
    check_paths(d, n_shapes, b.n_pods)
    n = _regime(ref, b, over)
    print(f"{route} {inst}: {d} over={len(over)} whole-GPU wins above totals={n}")
    assert n > 0, "no whole-GPU pod won on a node above its totals"


# ------------------------------------------------------------------------------------------------ the int32 guard
def _guard_cluster(rng, n_nodes):
    """mem_total 2^25 on every node; per GPU: free at its totals, just above them, or anywhere up to the guard.  Every
    4th node has two free GPUs and one at (2^20, 2^25): a k = 0 shape scores (2^25 + 2^20) / 2 * 100 there."""
    nodes = []
    for n in range(n_nodes):
        g = int(rng.choice([2, 4, 8]))
        core, mem = [], []
        for gi in range(g):
            k = int(rng.integers(0, 4))
            c, m = [(100, MAX_MEM), (100 + int(rng.integers(0, 3)), MAX_MEM - int(rng.integers(0, 3))),
                    (int(rng.integers(0, MAX_CORE + 1)), int(rng.integers(0, MAX_MEM + 1))),
                    (int(rng.choice([0, MAX_CORE])), int(rng.choice([0, MAX_MEM])))][k]
            core.append(c); mem.append(m)
        if n % 4 == 0 and g >= 4:
            core[:3], mem[:3] = [100, 100, MAX_CORE], [MAX_MEM, MAX_MEM, MAX_MEM]
        nodes.append((g, MAX_MEM, (core, mem)))
    return nodes


def _guard_shapes(rng):
    """k = 0 shapes (whole-GPU containers of count >= 2 only), single fractional containers up to the guard (the fast
    path), and multi-container shapes with large requests (general pods, the leaf-parallel Trade)."""
    big = lambda: (int(rng.choice([0, 1, MAX_CORE // 3, MAX_CORE])), int(rng.choice([1, MAX_MEM // 5, MAX_MEM // 2, MAX_MEM])), 0)
    shapes = [((0, 0, 2),), ((0, 0, 2), (0, 0, 2)), ((0, 0, 3),), ((0, 0, 4),)]
    while len(shapes) < 14:
        sh = (big(),) if len(shapes) < 9 else tuple(big() for _ in range(int(rng.integers(2, 4))))
        if sh not in shapes:
            shapes.append(sh)
    return shapes


@pytest.mark.parametrize("policy", [0, 1])
def test_int32_guard_limits(policy):
    """Rows up to (2^20, 2^25), requests up to the guard, k = 0 shapes.  Batch 1 holds only single fractional
    shapes (a monotone round set: cold evaluate, select, fast pods); batch 2 every shape (general pods and the
    leaf-parallel Trade on the same state).  Outputs, rows and caches (option_dump scores) against the oracle; RESCAN
    and schedule_batch_vec element for element.  Under binpack the largest score seen must pass 1.5e9."""
    cap = egs().capi
    rng = np.random.default_rng(2 ** 25 + policy)
    cl = Cluster(policy, _guard_cluster(rng, 300))
    shapes = _guard_shapes(rng)
    singles = [i for i, s in enumerate(shapes) if len(s) == 1 and s[0][2] == 0]
    picks = [np.array([singles[int(i)] for i in rng.integers(0, len(singles), 600)], np.int64),
             np.concatenate([np.arange(len(shapes)), rng.integers(0, len(shapes), 600)]).astype(np.int64)]
    o, e, r, v = cl.oracle(), cl.handle(), cl.handle(), cl.handle()
    ev0 = e.profile_get(cap.EGS_K_EVALUATE)[0]
    top, uid = 0, UID_BATCH
    for k, pick in enumerate(picks):
        b = Batch(policy, cl.nodes, shapes, pick)
        uids = np.arange(uid, uid + b.n_pods, dtype=np.uint64)
        uid += b.n_pods
        n_vec = 64
        ref = o.schedule_batch(b.c_off, b.units.astype(np.int64), uids=uids, threads=4, vec_pods=n_vec)
        compare_outputs(ref, e.schedule_batch(b.c_off, b.units, uids=uids, mode=cap.EGS_MODE_ROUNDS), f"rounds batch {k}")
        compare_outputs(ref, r.schedule_batch(b.c_off, b.units, uids=uids, mode=cap.EGS_MODE_RESCAN), f"rescan batch {k}")
        got = v.schedule_batch_vec(b.c_off, b.units, n_vec, uids=uids)
        compare_outputs(ref, got, f"vec batch {k}")
        assert np.array_equal(ref["vec_fit"], got["vec_fit"]), f"vec_fit batch {k}"
        fit = ref["vec_fit"] == 1
        assert np.array_equal(ref["vec_score"][fit], got["vec_score"][fit]), f"vec_score batch {k}"
        top = max(top, int(got["vec_score"][fit].max(initial=0)))
        compare_rows(e, o, range(len(cl.nodes)))
        compare_rows(r, o, range(len(cl.nodes)))
        compare_caches(e, o, distinct_shapes(b), range(len(cl.nodes)), unfit_check=True)
        for sh in distinct_shapes(b):
            st, sc, _ = e.option_dump(list(sh))
            top = max(top, int(sc[st == 1].max(initial=0)))
        if k == 0:
            assert e.profile_get(cap.EGS_K_EVALUATE)[0] - ev0 == len(singles)   # every shape cold: one evaluate each
    for h in (e, r, v):
        h.close()
    if policy == 0:
        assert top > 1.5e9, top
    else:
        assert top == 0, top


# ------------------------------------------------------------------------------------------------ sharded
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_above_totals_equal_unsharded(world):
    """The over-totals batch ("load" route, 64 shapes) on an in-process shard group (egs_comm_init_local, one thread
    per rank): every rank's outputs equal the unsharded run, every shard's rows the unsharded rows."""
    cl, b, _ = _over_case(7000 + world, "load", 64, n_nodes=400, n_pods=3000)
    ref, rows, ranks = run_sharded(cl.handle, world, b.c_off, b.units)
    compare_outputs(cl.oracle().schedule_batch(b.c_off, b.units.astype(np.int64), threads=4), ref, "unsharded")
    compare_shards(ref, rows, ranks, f"world {world}")
