"""egs_schedule_batch_nodes: candidate node sets per pod, against the oracle driven with the same node lists
(oracle_harness.oracle_batch with node_ids).  Every case compares the six per-pod outputs, the final rows of every node
and the option cache of every shape on every node, "known not to fit" marks included."""
import numpy as np
import pytest

from oracle_harness import Cluster, compare_caches, compare_outputs, compare_rows, egs, oracle_batch
from shard_groups import ShardGroup, hetero_nodes, mixed_shapes
import wave_clusters as wc

pytestmark = pytest.mark.gpu

RESCAN, ROUNDS = 1, 2
SENT = (-1, -1, 0)


def _batch(rng, shapes, n_pods):
    pick = rng.integers(0, len(shapes), n_pods)
    units = np.array([u for p in pick for u in shapes[p]], np.int32).reshape(-1, 3)
    c_off = np.concatenate([[0], np.cumsum([len(shapes[p]) for p in pick])]).astype(np.int32)
    return c_off, units


def _lists(sets, pod_set, P):
    ps = np.zeros(P, np.int32) if pod_set is None else pod_set
    ids = [np.flatnonzero(s).astype(np.int32) for s in sets]
    return [ids[ps[p]] for p in range(P)]


def _check(e, o, shapes, ref, got, what):
    compare_outputs(ref, got, what)
    compare_rows(e, o, range(e.max_nodes))
    compare_caches(e, o, shapes, range(e.max_nodes), unfit_check=True)


def _runs(P, run, n_sets):
    return (np.arange(P) // run % n_sets).astype(np.int32)


def _sets(rng, n_sets, n, density):
    return [rng.random(n) < density for _ in range(n_sets)]


# ------------------------------------------------------------------------------------------------ 1. all-ones set
@pytest.mark.parametrize("mode", [RESCAN, ROUNDS])
def test_all_ones_set_is_schedule_batch(mode):
    rng = np.random.default_rng(mode)
    cl = Cluster(0, hetero_nodes(rng, 300))
    shapes = mixed_shapes(rng, 24)
    c_off, units = _batch(rng, shapes, 500)
    a, b = cl.handle(), cl.handle()
    ref = a.schedule_batch(c_off, units, mode=mode)
    got = b.schedule_batch_nodes(c_off, units, [np.ones(cl.n_nodes, bool)], mode=mode)
    compare_outputs(ref, got, "all-ones set")
    for x, y in zip(a.state_dump(), b.state_dump()):
        assert np.array_equal(x, y)
    for sh in shapes:
        for x, y in zip(a.option_dump(list(sh)), b.option_dump(list(sh))):
            assert np.array_equal(x, y), f"shape {sh}: caches differ"
    assert b.pod_known(0x8000000000000000 + int(np.flatnonzero(got["status"] == 0)[0]))   # library-assigned uids


# ------------------------------------------------------------------------------------------------ 2. random sets
@pytest.mark.parametrize("density", [0.05, 0.5, 0.95])
@pytest.mark.parametrize("run", [1, 7, 300, 0])
@pytest.mark.parametrize("kind", ["rescan", "rounds", "rounds_host_sets"])
def test_random_sets_8_wide(kind, run, density):
    rng = np.random.default_rng([run, int(density * 100), len(kind)])
    cl = Cluster(run & 1, hetero_nodes(rng, 260))
    shapes = mixed_shapes(rng, 120 if kind == "rounds_host_sets" else 20)
    P = 600
    c_off, units = _batch(rng, shapes, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    sets = _sets(rng, 3, cl.n_nodes, density)
    pod_set = _runs(P, run or P, len(sets))
    e, o = cl.handle(), cl.oracle()
    got = e.schedule_batch_nodes(c_off, units, sets, pod_set, uids, mode=RESCAN if kind == "rescan" else ROUNDS)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists(sets, pod_set, P))
    _check(e, o, shapes, ref, got, f"{kind} run {run} density {density}")


@pytest.mark.parametrize("density", [0.05, 0.5, 0.95])
@pytest.mark.parametrize("run", [1, 7, 300, 0])
def test_random_sets_wide(run, density):
    rng = np.random.default_rng([16, run, int(density * 100)])
    nodes = []
    for _ in range(120):
        g = int(rng.choice([2, 8, 12, 16]))
        core = [int(rng.choice([100, 100, 60, 0])) for _ in range(g)]
        nodes.append((g, 64, (core, [64 if c == 100 else int(rng.integers(0, 65)) for c in core])))
    cl = Cluster(run & 1, nodes, g_max=16)
    shapes = [((30, 8, 0),), ((0, 0, 1),), ((0, 0, 10),), ((20, 4, 0), (0, 0, 2)), ((50, 16, 0), SENT)]
    P = 400
    c_off, units = _batch(rng, shapes, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    sets = _sets(rng, 2, cl.n_nodes, density)
    pod_set = _runs(P, run or P, 2)
    e, o = cl.handle(), cl.oracle()
    got = e.schedule_batch_nodes(c_off, units, sets, pod_set, uids)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists(sets, pod_set, P))
    _check(e, o, shapes, ref, got, f"wide run {run} density {density}")


@pytest.mark.parametrize("density", [0.05, 0.5, 0.95])
@pytest.mark.parametrize("run", [1, 7, 300, 0])
def test_random_sets_sidecar(run, density):
    rng = np.random.default_rng([8, run, int(density * 100)])
    nodes = []
    for _ in range(48):
        g = int(rng.integers(1, 9))
        core = [int(rng.choice([100, 100, 60, 0])) for _ in range(g)]
        nodes.append((g, 32, (core, [32 if c == 100 else int(rng.integers(0, 33)) for c in core])))
    cl = Cluster(run & 1, nodes, c_max=8)
    split = ((10, 2, 0), SENT, SENT, SENT, SENT, (0, 0, 1))         # 5 branching on 8 GPUs: the leaf-split Trade
    shapes = [split, ((20, 4, 0), SENT, SENT), ((0, 0, 1),), ((0, 0, 1), SENT, SENT, SENT, SENT, SENT, (5, 1, 0))]
    P = 120
    c_off, units = _batch(rng, shapes, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    sets = _sets(rng, 2, cl.n_nodes, density)
    pod_set = _runs(P, run or P, 2)
    e, o = cl.handle(), cl.oracle()
    got = e.schedule_batch_nodes(c_off, units, sets, pod_set, uids)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists(sets, pod_set, P), planes=8)
    _check(e, o, shapes, ref, got, f"sidecar run {run} density {density}")


# ------------------------------------------------------------------------------------------------ 3. stale caches
@pytest.mark.parametrize("mode", [RESCAN, ROUNDS])
def test_excluded_node_keeps_its_stale_option(mode):
    rng = np.random.default_rng(33)
    cl = Cluster(0, [(8, 64, None) for _ in range(64)])
    shapes = [((20, 4, 0),), ((0, 0, 1), (10, 2, 0))]
    e, o = cl.handle(), cl.oracle()
    c_off, units = _batch(rng, shapes, 40)
    uids = np.arange(1, 41, dtype=np.uint64)
    every = np.ones(64, bool)
    got = e.schedule_batch_nodes(c_off, units, [every], uids=uids, mode=mode)      # every node caches both shapes
    compare_outputs(oracle_batch(o, c_off, units, uids, node_ids=_lists([every], None, 40)), got, "warm-up")
    before = [e.option_dump(list(sh)) for sh in shapes]
    X = int(np.flatnonzero((before[0][0] == 1) & (before[1][0] == 1))[0])   # a node caching both shapes
    no_x = every.copy(); no_x[X] = False
    c_off, units = _batch(rng, shapes, 60)
    uids = np.arange(100, 160, dtype=np.uint64)
    got = e.schedule_batch_nodes(c_off, units, [no_x], uids=uids, mode=mode)
    compare_outputs(oracle_batch(o, c_off, units, uids, node_ids=_lists([no_x], None, 60)), got, "X excluded")
    for sh, b in zip(shapes, before):
        for x, y in zip(b, e.option_dump(list(sh))):
            assert np.array_equal(x[X], y[X]), f"shape {sh}: the option of the excluded node changed"
    rec = (0, X, [(30, 8, 0)], [[0]], 999)                          # AddPod on X voids no cache entry
    assert e.mutations_apply([rec]) == 0
    o.add_pod(X, [(30, 8, 0)], [[0]], 999)
    c_off, units = _batch(rng, shapes, 60)
    uids = np.arange(200, 260, dtype=np.uint64)
    got = e.schedule_batch_nodes(c_off, units, [every], uids=uids, mode=mode)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists([every], None, 60))
    _check(e, o, shapes, ref, got, "X admitted again")


# ------------------------------------------------------------------------------------------------ 4. cold shapes
def test_cold_shapes_leave_excluded_nodes_absent():
    rng = np.random.default_rng(4)
    cl = Cluster(1, hetero_nodes(rng, 200))
    shapes = mixed_shapes(rng, 10)
    e, o = cl.handle(), cl.oracle()
    e.snapshot()
    c_off, units = _batch(rng, shapes, 50)
    e.schedule_batch(c_off, units, mode=ROUNDS)
    e.restore()                                                      # the loaded rows, every option table cold
    s = rng.random(cl.n_nodes) < 0.5
    c_off, units = _batch(rng, shapes, 200)
    uids = np.arange(1, 201, dtype=np.uint64)
    got = e.schedule_batch_nodes(c_off, units, [s], uids=uids, mode=ROUNDS)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists([s], None, 200))
    _check(e, o, shapes, ref, got, "cold shapes")
    for sh in shapes:
        st = e.option_dump(list(sh))[0]
        assert (st[~s] == 0).all(), f"shape {sh}: an excluded node left OPT_ABSENT"


# ------------------------------------------------------------------------------------------------ 5. shard groups
@pytest.mark.parametrize("world", [2, 4, 8])
def test_shard_group(world):
    rng = np.random.default_rng(world)
    n = 128 * 2 * world + 37
    cl = Cluster(world & 1, hetero_nodes(rng, n))
    shapes = mixed_shapes(rng, 16)
    P = 400
    c_off, units = _batch(rng, shapes, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    cap = egs().capi
    lo1, hi1 = cap.shard_range(n, 1, world)
    only_first = np.zeros(n, bool); only_first[:lo1] = rng.random(lo1) < 0.7     # empty on every rank but rank 0
    inside = np.zeros(n, bool); inside[lo1 + 50:hi1 - 20] = True                   # boundaries inside shard 1
    sets = [only_first, inside, rng.random(n) < 0.3]
    pod_set = _runs(P, 13, 3)
    e, o = cl.handle(), cl.oracle()
    twin = e.schedule_batch_nodes(c_off, units, sets, pod_set, uids, mode=ROUNDS)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists(sets, pod_set, P))
    _check(e, o, shapes, ref, twin, f"world {world}, unsharded")
    with ShardGroup(cl, world) as g:
        outs = g.each(lambda r, h: h.schedule_batch_nodes(c_off, units, sets, pod_set, uids, mode=ROUNDS))
        for r, out in enumerate(outs):
            compare_outputs(twin, out, f"world {world}, rank {r}")

        for r in range(world):
            def check(_, h, own=list(g.own(r))):
                if own:
                    compare_rows(h, o, own)
                    compare_caches(h, o, shapes, own, unfit_check=True)
            g.on(r, check)


# ------------------------------------------------------------------------------------------------ 6. wave clusters
def test_wave_cluster_chunk_edges():
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    n = wc.wave(n_sm) + 300                                           # more chunks than one k_select wave holds
    rng = np.random.default_rng(6)
    core = np.full((n, 8), 100, np.int32); mem = np.full((n, 8), 80, np.int32)
    core[rng.random((n, 8)) < 0.3] = 40
    cl = wc.rows_cluster(0, core, mem)
    shapes = [((30, 8, 0),), ((0, 0, 2),), ((50, 40, 0), (0, 0, 1))]
    P = 300
    c_off, units = _batch(rng, shapes, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    edges = np.zeros(n, bool)
    for c in range(0, n, 128):                                        # the last and the first node of every chunk
        edges[c] = True
        edges[min(c + 127, n - 1)] = True
    W = wc.wave(n_sm) // 128
    across = np.zeros(n, bool); across[(W - 4) * 128:(W + 2) * 128] = True       # chunks on both sides of the wave
    ends = np.zeros(n, bool); ends[:4 * 128] = True; ends[(W + 2) * 128:] = True  # its complement's ends
    sets = [edges, across, ends]
    pod_set = _runs(P, 50, 3)
    e, o = cl.handle(), cl.oracle()
    got = e.schedule_batch_nodes(c_off, units, sets, pod_set, uids, mode=ROUNDS)
    ref = oracle_batch(o, c_off, units, uids, node_ids=_lists(sets, pod_set, P))
    compare_outputs(ref, got, "wave cluster")
    touched = set(int(x) for x in ref["node"] if x >= 0) | set(range(0, n, 97))
    compare_rows(e, o, touched)
    compare_caches(e, o, shapes, sorted(touched), unfit_check=True)


# ------------------------------------------------------------------------------------------------ 7. empty and malformed
@pytest.mark.parametrize("mode", [RESCAN, ROUNDS])
def test_empty_set_and_malformed_arguments(mode):
    rng = np.random.default_rng(7)
    cl = Cluster(0, hetero_nodes(rng, 100))
    shapes = mixed_shapes(rng, 6)
    e = cl.handle()
    c_off, units = _batch(rng, shapes, 30)
    e.schedule_batch(c_off, units, mode=mode)
    cap = egs().capi

    def state():
        return [x.copy() for x in e.state_dump()] + [x.copy() for sh in shapes for x in e.option_dump(list(sh))]

    def same(a, b):
        return all(np.array_equal(x, y) for x, y in zip(a, b))
    s0 = state()
    uids = np.arange(1000, 1030, dtype=np.uint64)
    got = e.schedule_batch_nodes(c_off, units, [np.zeros(100, bool)], uids=uids, mode=mode)
    assert (got["status"] == cap.EGS_ERR_NOFIT).all() and (got["fit_count"] == 0).all() and (got["node"] == -1).all()
    assert same(s0, state())
    assert not any(e.pod_known(int(u)) for u in uids)

    words = cap.node_set_words(100)
    good = cap.node_sets_array([np.ones(100, bool)], 100)
    beyond = good.copy(); beyond[0, words - 1] |= np.uint64(1) << np.uint64(100 % 64)
    c_off32 = np.ascontiguousarray(c_off, np.int32); units32 = np.ascontiguousarray(units, np.int32)
    out = np.zeros(30, np.int32)
    P = len(c_off) - 1

    def call(n_sets, sets, pod_set):
        return e.L.egs_schedule_batch_nodes(e.h, mode, P, cap._p(c_off32), cap._p(units32), None, n_sets,
                                            cap._p(sets), cap._p(pod_set), cap._p(out), None, None, None, None, None)
    bad_ps = np.zeros(P, np.int32); bad_ps[-1] = 1
    neg_ps = np.zeros(P, np.int32); neg_ps[3] = -1
    for what, rc in [("n_sets 0", call(0, good, None)), ("sets NULL", call(1, None, None)),
                     ("pod_set out of range", call(1, good, bad_ps)), ("pod_set negative", call(1, good, neg_ps)),
                     ("bit beyond max_nodes", call(1, beyond, None))]:
        assert rc == cap.EGS_ERR_BAD_ARG, what
        assert same(s0, state()), f"{what}: something was applied"


# ------------------------------------------------------------------------------------------------ 8. checkpoint
def test_checkpoint_rollback_and_library_uids():
    rng = np.random.default_rng(8)
    cl = Cluster(1, hetero_nodes(rng, 300))
    shapes = mixed_shapes(rng, 12)
    e = cl.handle()
    P = 300
    c_off, units = _batch(rng, shapes, P)
    sets = _sets(rng, 3, cl.n_nodes, 0.6)
    pod_set = _runs(P, 40, 3)
    e.checkpoint_save()
    s0 = [x.copy() for x in e.state_dump()] + [x.copy() for sh in shapes for x in e.option_dump(list(sh))]
    first = e.schedule_batch_nodes(c_off, units, sets, pod_set, mode=ROUNDS)
    base = 0x8000000000000000
    for p in range(P):                                                # library uids run on across the runs
        assert e.pod_known(base + p) == (first["status"][p] == 0), f"pod {p}"
    e.checkpoint_rollback()
    s1 = [x.copy() for x in e.state_dump()] + [x.copy() for sh in shapes for x in e.option_dump(list(sh))]
    assert all(np.array_equal(x, y) for x, y in zip(s0, s1)), "rollback is not exact"
    again = e.schedule_batch_nodes(c_off, units, sets, pod_set, mode=ROUNDS)
    compare_outputs(first, again, "rerun after rollback")
    o = cl.oracle()
    ref = oracle_batch(o, c_off, units, np.arange(base, base + P, dtype=np.uint64), node_ids=_lists(sets, pod_set, P))
    _check(e, o, shapes, ref, again, "checkpoint rerun")
