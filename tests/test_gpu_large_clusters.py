"""Every engine and verb on clusters larger than one k_select wave (tests/wave_clusters.py): past wave(n_sm) nodes per
shard a k_select warp carries its top-32 lists and aggregates from one 128-node chunk to the next, k_merge folds the
lists of a full grid, and k_pass folds thousands of partials.  Sizes follow the device's SM count, and every test
asserts that the shards it runs give some warp at least two chunks, so a part with more SMs grows the sizes instead of
losing the coverage.  The planted cases are compared with the C oracle; at 10^6 nodes and more the engines are checked
against each other."""
import os

import numpy as np
import pytest

from oracle_harness import Cluster, compare_caches, compare_outputs, compare_rows, compare_shards, conservation, egs, \
    late_window, run_sharded
from wave_clusters import CASES, case_a, case_d, chunks_per_warp, sizes, wave

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 4
MODES = {"rescan": 1, "rounds": 2}


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _past_wave(n_nodes, n_sm, world=1):
    """Every shard of n_nodes nodes at `world` gives warp 0 of k_select at least two chunks; returns the shards."""
    shards = [egs().capi.shard_range(n_nodes, r, world) for r in range(world)]
    for r, (lo, hi) in enumerate(shards):
        assert hi - lo > wave(n_sm) and chunks_per_warp(hi - lo, n_sm) >= 2, (n_nodes, world, r, lo, hi)
        assert r == 0 or lo != 0
    return shards


def _sample(n_nodes, seed, k=2000):
    return set(int(x) for x in np.random.default_rng(seed).integers(0, n_nodes, k))


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("case", list(CASES))
def test_planted_case_vs_oracle(n_sm, case, policy):
    """Planted case x policy x {rescan, rounds} at W + 1 and 2W + 127 nodes: the six per-pod outputs, the rows of every
    touched node, of the nodes around the wave and of a seeded sample, and the option caches of the batch's shapes on
    those nodes (with the "does not fit" memos) equal the oracle's."""
    for N in sizes(n_sm):
        _past_wave(N, n_sm)
        p = CASES[case](N, n_sm, policy)
        o = p.cluster.oracle()
        ref = o.schedule_batch(p.c_off, p.units.astype(np.int64), threads=THREADS)
        assert (ref["status"] == 0).any()
        W = wave(n_sm)
        nodes = _sample(N, N) | set(range(W - 64, min(N, W + 64))) | set(range(N - 32, N)) \
            | set(int(x) for x in ref["node"] if x >= 0)
        for name, mode in MODES.items():
            e = p.cluster.handle()
            compare_outputs(ref, e.schedule_batch(p.c_off, p.units, mode=mode), f"{p.name} N={N} {name}")
            compare_rows(e, o, nodes)
            compare_caches(e, o, p.shapes, nodes, unfit_check=True)
            e.close()


@pytest.mark.parametrize("case,policy,vec_pods", [("D40", 0, 8), ("B", 1, 6), ("A", 0, 4)])
def test_full_vectors_past_the_wave(n_sm, case, policy, vec_pods):
    """The full per-pod fit mask and score vector of the first pods equal the oracle's element-wise."""
    for N in sizes(n_sm):
        _past_wave(N, n_sm)
        p = CASES[case](N, n_sm, policy, n_pods=vec_pods)
        ref = p.cluster.oracle().schedule_batch(p.c_off, p.units.astype(np.int64), threads=THREADS, vec_pods=vec_pods)
        got = p.cluster.handle().schedule_batch_vec(p.c_off, p.units, vec_pods)
        compare_outputs(ref, got, f"{p.name} N={N}")
        assert np.array_equal(ref["vec_fit"], got["vec_fit"]), f"{p.name} N={N}: fit vector"
        assert np.array_equal(ref["vec_score"], got["vec_score"]), f"{p.name} N={N}: score vector"
        assert got["vec_fit"][:, wave(n_sm):].any()


def test_late_window_past_the_wave(n_sm):
    """config 4 at 3W nodes, scheduled on the GPU to 90 % of config 4's batch (10 pods per node); then a fresh oracle
    loaded with the rows and every cache and the GPU schedule the next 200 pods and must agree on every output, the
    rows and the caches."""
    N = 3 * wave(n_sm)
    _past_wave(N, n_sm)
    K = 9 * N
    ref, e = late_window(4, None, K, 200, n_nodes=N, threads=THREADS, sample=1500)
    core = e.state_dump()[0][:, :8]
    w = egs().workloads.config(4, n_nodes=N, n_pods=1)
    used = 1 - core.sum() / (100 * core.size)
    assert used > 1 - w.core.sum() / (100 * core.size) + 0.15         # the prefix filled the cluster
    assert (ref["status"] == 0).any()


def test_verbs_over_million_ids(n_sm):
    """filter / score on a handle of at least 2^20 nodes over seeded permutations with duplicates and out-of-range ids,
    4 096 -> 10^5 -> 10^6 ids long (the gather and staging buffers grow between calls), against the oracle; then the
    option cache of every shape used on a sample."""
    N = max(1 << 20, 3 * wave(n_sm))
    _past_wave(N, n_sm)
    w = egs().workloads.config(4, n_nodes=N, n_pods=2000)
    cl = Cluster.of_workload(w)
    e, o = cl.handle(), cl.oracle()
    shapes = egs().workloads.shapes_of(w)[:3]
    rng = np.random.default_rng(7)
    for L, sh in zip([4096, 100_000, 1_000_000], shapes):
        ids = rng.permutation(N)[:L].astype(np.int32)
        k = L // 16
        ids[rng.integers(0, L, k)] = ids[rng.integers(0, L, k)]                        # duplicates
        ids[rng.integers(0, L, 8)] = rng.choice([-1, -7, N, N + 5, 1 << 30], 8)          # out of range
        req = list(sh)
        fit = o.filter(ids, req)        # one oracle worker: two workers would fill a duplicate node's cache at once
        got = e.filter(ids, req)
        bad = np.nonzero(fit != got)[0]
        assert bad.size == 0, f"L={L}: filter differs at ids {ids[bad[:5]].tolist()}"
        assert fit.sum() > 0
        st_o, sc_o = o.score(ids, req)
        st_e, sc_e = e.score(ids, req)
        assert st_o == st_e == 0
        bad = np.nonzero(sc_o != sc_e)[0]
        assert bad.size == 0, f"L={L}: score differs at ids {ids[bad[:5]].tolist()}"
    nodes = _sample(N, 8, 3000) | set(int(i) for i in ids[:500] if 0 <= i < N)
    compare_caches(e, o, shapes, nodes, unfit_check=True)
    compare_rows(e, o, nodes)


@pytest.mark.parametrize("which", ["cfg4", "D110"])
def test_engines_agree_at_a_million_nodes(n_sm, which):
    """No oracle at this size: the rounds engine, the per-pod rescan engine and the per-pod engine on a wide handle
    (g_max 16, k_pass<16>) over the same 8-GPU cluster agree on every output and on the rows after 10^5 pods; on
    config 4 the rows are also what the binds leave.  (Planted case D has multi-container pods whose failing binds keep
    their earlier Adds, gpu.go Transact, so its rows cannot be rebuilt from the outputs alone.)"""
    N = max(1 << 20, 8 * wave(n_sm))
    _past_wave(N, n_sm)
    P = 100_000
    if which == "cfg4":
        w = egs().workloads.config(4, n_nodes=N, n_pods=P)
        cl, c_off, units = Cluster.of_workload(w), w.c_off, w.units
    else:
        p = case_d(N, n_sm, 0, n_shapes=110, n_pods=P)
        cl, c_off, units = p.cluster, p.c_off, p.units
    outs, rows = {}, {}
    for name, mode, g_max in [("rounds", 2, 8), ("rescan", 1, 8), ("wide", 1, 16)]:
        e = Cluster.of_workload(cl.workload, g_max).handle()
        outs[name] = e.schedule_batch(c_off, units, mode=mode)
        rows[name] = e.state_dump()[:2]
        if which == "cfg4":
            conservation(w, outs[name], e)
        e.close()
    ref = outs["rounds"]
    assert (ref["status"] == 0).sum() > (P // 2 if which == "cfg4" else 0)
    for name in ("rescan", "wide"):
        compare_outputs(ref, outs[name], f"{which}: {name} against rounds")
        for a, b in zip(rows["rounds"], rows[name]):
            assert np.array_equal(a, b[:, :8]), f"{which}: rows of {name} against rounds"
        assert name != "wide" or (rows[name][0][:, 8:] == egs().capi.EGS_PAD).all()


@pytest.mark.parametrize("world,extra", [(2, 300), (4, 1024)])
def test_shard_groups_past_the_wave(n_sm, world, extra):
    """In-process shard groups where every shard is larger than a wave (N = world * W + extra; 4W + 300 would leave
    rank 0 exactly W nodes, since shard cuts round down to multiples of 128): planted case A and config 4 on every rank
    equal the unsharded run; the unsharded run of case A and its rows equal the oracle's."""
    N = world * wave(n_sm) + extra
    _past_wave(N, n_sm, world)
    p = case_a(N, n_sm, 0)
    ref, rows, ranks = run_sharded(p.cluster.handle, world, p.c_off, p.units)
    compare_shards(ref, rows, ranks, f"case A world {world}")
    o = p.cluster.oracle()
    compare_outputs(o.schedule_batch(p.c_off, p.units.astype(np.int64), threads=THREADS), ref, f"case A N={N}")
    nodes = np.unique(np.concatenate([np.arange(N - 256, N), ref["node"][ref["node"] >= 0],
                                      np.arange(wave(n_sm) - 64, wave(n_sm) + 64)]))
    ocore, omem, _ = o.rows_many(nodes, 8)
    assert np.array_equal(rows[0][nodes, :8], ocore) and np.array_equal(rows[1][nodes, :8], omem), "case A: rows"
    w = egs().workloads.config(4, n_nodes=N, n_pods=30_000)
    ref, rows, ranks = run_sharded(Cluster.of_workload(w).handle, world, w.c_off, w.units)
    compare_shards(ref, rows, ranks, f"cfg4 world {world}")
    assert (ref["status"] != 1).all()         # room for every pod; status 3 (a stale cached option) is reference behaviour
