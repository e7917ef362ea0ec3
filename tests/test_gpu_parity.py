"""Parity tests proper: libegs (CUDA, through the C ABI) against the oracle, bit-exact."""
import numpy as np
import pytest

import oracle_c as oc
from ka_vectors import KA0_FINAL, KA0_MEM, KA0_TRACE, TRADE_KA
from oracle_harness import Cluster, compare_caches, compare_outputs, compare_rows, egs
from scenario import CBackend, GpuBackend, make_scenario, run_scenario

pytestmark = pytest.mark.gpu

KA0_CLUSTER = Cluster(0, [(2, 16, None)] * 4)          # config 0: four nodes of two 16 MiB GPUs, binpack


@pytest.mark.parametrize("name,policy,mt,rows,req,exp", TRADE_KA, ids=[k[0] for k in TRADE_KA])
def test_trade_ka_gpu(name, policy, mt, rows, req, exp):
    e = egs().Egs(policy, 4)
    assert e.node_set(0, len(rows), mt) == 0
    assert e.state_load(0, [r[0] for r in rows], [r[1] for r in rows]) == 0
    fit = e.filter([0], req)
    assert bool(fit[0]) == (exp is not None)
    assert e.peek(0, req) == exp
    assert e.rows(0) == list(rows)


@pytest.mark.parametrize("mode", [1, 2])
def test_ka0_batch(mode):
    w = egs().workloads.config(0)
    e = KA0_CLUSTER.handle()
    out = e.schedule_batch(w.c_off, w.units, mode=mode)
    for p, (fit, scores, node, status, alloc) in enumerate(KA0_TRACE):
        assert out["node"][p] == node and out["status"][p] == status and out["fit_count"][p] == sum(fit)
        assert egs().capi.masks_to_lists(out["alloc_mask"][p], 1) == [alloc[0] if alloc else []]
    assert [e.rows(i) for i in range(4)] == KA0_FINAL
    assert e.pod_known(0x8000000000000000 + 6) and not e.pod_known(0x8000000000000000 + 7)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", range(30))
def test_scenarios_gpu_vs_oracle(seed, policy):
    nodes, ops = make_scenario(seed * 2 + policy, max_c=4 if seed % 3 == 0 else 3)
    a = run_scenario(CBackend(policy), nodes, ops, policy)
    b = run_scenario(GpuBackend(policy), nodes, ops, policy)
    assert a == b


def _compare_batch(w, mode, threads=1):
    cl = Cluster.of_workload(w)
    o = cl.oracle()
    ref = o.schedule_batch(w.c_off, w.units64(), threads=threads)
    e = cl.handle()
    got = e.schedule_batch(w.c_off, w.units, mode=mode)
    compare_outputs(ref, got, f"config {w.cfg} mode {mode}")
    compare_rows(e, o, range(w.n_nodes))
    return ref, got, e, o


@pytest.mark.parametrize("mode", [1, 2])
def test_cfg1_full(mode):
    """BASELINE config 1 at full size: 1000 nodes x 8 GPUs, 10000 pods, binpack."""
    _compare_batch(egs().workloads.config(1), mode)


@pytest.mark.parametrize("mode", [1, 2])
def test_cfg2_prefix(mode):
    """config 2 (spread, core+memory): 10000 nodes, first 20000 pods against the oracle."""
    _compare_batch(egs().workloads.config(2, n_pods=20000), mode, threads=4)


@pytest.mark.parametrize("policy", [1, 0])
@pytest.mark.parametrize("mode", [1, 2])
def test_cfg3_multi_container_prefix(mode, policy):
    """config 3 (2-3 containers per pod): 50000 nodes, first 1500 pods, spread as named + binpack."""
    _compare_batch(egs().workloads.config(3, n_pods=1500, policy=policy), mode)


@pytest.mark.parametrize("mode", [1, 2])
def test_cfg4_prefix(mode):
    """config 4: 100000 nodes, first 3000 pods against the oracle (4-worker filter like scheduler.go:135)."""
    _compare_batch(egs().workloads.config(4, n_pods=3000), mode, threads=4)


def _late_window(cfg, policy, K, W, threads=4, sample=4000):
    """The GPU engine schedules the first K pods; rows and every option cache are dumped through the ABI and
    loaded into a FRESH oracle (egso_cache_load); both then schedule pods [K, K+W) and must agree on all six
    outputs, the final rows and the final caches.  This puts the oracle into the late, full-cluster regime
    (stale options, bind failures, unfit nodes) that a prefix from an empty cluster never reaches."""
    eg = egs()
    full = eg.workloads.config(cfg, n_pods=K + W, policy=policy)
    e = Cluster.of_workload(full).handle()
    pre = full.prefix(K)
    e.schedule_batch(pre.c_off, pre.units, mode=2)
    core, mem, _, _ = e.state_dump()
    o = oc.OracleC(full.policy)
    for n in range(full.n_nodes):
        o.add_node(100 * full.gpus, full.mem_total * full.gpus)
        o.set_rows(n, core[n, :full.gpus], mem[n, :full.gpus])
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
    return ref


@pytest.mark.parametrize("K", [250_000, 500_000, 750_000, 900_000, 990_000])
def test_cfg4_late_windows(K):
    """config 4 at full size, 3000-pod windows deep inside the 1M-pod batch (incl. the > 80 % regime)."""
    _late_window(4, None, K, 3000)


@pytest.mark.parametrize("K", [100_000, 400_000])
def test_cfg3_late_windows(K):
    _late_window(3, None, K, 1500)


@pytest.mark.parametrize("K", [50_000, 90_000])
def test_cfg2_late_windows(K):
    _late_window(2, None, K, 5000)


@pytest.mark.parametrize("cfg,n_pods,vec_pods", [(0, None, 8), (1, 10000, 1500), (2, 3000, 600)])
def test_full_fit_and_score_vectors(cfg, n_pods, vec_pods):
    """SURVEY 8d: on configs 0-2 the FULL per-pod fit mask and score vector (what /scheduler/filter and
    /scheduler/priorities return for every candidate node) are compared element-wise with the oracle."""
    w = egs().workloads.config(cfg, n_pods=n_pods)
    cl = KA0_CLUSTER if cfg == 0 else Cluster.of_workload(w)
    e, o = cl.handle(), cl.oracle()
    ref = o.schedule_batch(w.c_off, w.units64(), vec_pods=vec_pods)
    got = e.schedule_batch_vec(w.c_off, w.units, vec_pods)
    compare_outputs(ref, got, f"config {cfg}")
    assert np.array_equal(ref["vec_fit"], got["vec_fit"])
    assert np.array_equal(ref["vec_score"], got["vec_score"])
    assert got["vec_fit"].sum() > 0


def test_pressure_small_cluster():
    """Few nodes, many pods: nodes fill up, unfit nodes and stale-option bind failures appear."""
    eg = egs()
    for cfg, pol in [(1, 0), (2, 1), (4, 0), (3, 1), (3, 0)]:
        w = eg.workloads.config(cfg, n_nodes=40, n_pods=4000, policy=pol)
        for mode in (1, 2):
            ref, got, _, _ = _compare_batch(w, mode)
        assert (ref["status"] == 3).sum() + (ref["status"] == 1).sum() > 0, "scenario must exercise failures"


def _conservation(w, out, e):
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


@pytest.mark.parametrize("cfg", [2, 4])
def test_full_size_properties(cfg):
    """Full BASELINE sizes (cfg2: 10k nodes/100k pods; cfg4: 100k nodes/1M pods): the two
    independent device loops (per-pod rescan, rounds) agree on every output, and resources are conserved."""
    w = egs().workloads.config(cfg)
    cl = Cluster.of_workload(w)
    a = cl.handle().schedule_batch(w.c_off, w.units, mode=1)
    e2 = cl.handle()
    b = e2.schedule_batch(w.c_off, w.units, mode=2)
    compare_outputs(a, b, f"config {cfg} rounds against rescan")
    _conservation(w, b, e2)
    assert (b["status"] != 1).all()   # the named clusters have room for every pod (no NOFIT);
    # status 3 (stale cached option, gpu.go:158-168) is reference behaviour and does occur under spread


def _random_batch(seed, n_nodes, n_pods, n_shapes, policy):
    """Mixed shapes: fractional, whole-GPU (count 1..2), -1 sentinel containers, 1..4 containers per pod;
    heterogeneous nodes (G in 1,2,4,8).  Non-monotone rounds: sentinel units ADD 1 to a GPU (gpu.go:36-37)."""
    rng = np.random.default_rng(seed)
    nodes = []
    for n in range(n_nodes):
        g = int(rng.choice([1, 2, 4, 8]))
        m = int(rng.choice([16, 40, 80]))
        rows = None
        if rng.integers(0, 2):
            rows = ([int(rng.choice([100, 100, 60, 30, 0])) for _ in range(g)], [int(rng.integers(0, m + 1)) for _ in range(g)])
        nodes.append((g, m, rows))
    shapes = []
    for _ in range(n_shapes):
        c = int(rng.integers(1, 5))
        units = []
        for _ in range(c):
            k = rng.integers(0, 10)
            if k == 0:
                units.append((-1, -1, 0))
            elif k == 1:
                units.append((0, 0, int(rng.integers(1, 3))))
            else:
                units.append((int(rng.choice([0, 5, 10, 25, 50])), int(rng.integers(1, 12)), 0))
        shapes.append(units)
    pick = rng.integers(0, n_shapes, n_pods)
    c_off = [0]
    units = []
    for s in pick:
        units.extend(shapes[int(s)])
        c_off.append(len(units))
    return Cluster(policy, nodes), np.array(c_off, np.int32), np.array(units, np.int32)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed,n_nodes,n_pods,n_shapes", [(1, 50, 3000, 6), (2, 300, 4000, 12), (3, 2000, 3000, 40), (4, 20, 2000, 3)])
def test_batch_mixed_shapes_vs_oracle(seed, n_nodes, n_pods, n_shapes, policy):
    cl, c_off, units = _random_batch(seed, n_nodes, n_pods, n_shapes, policy)
    for mode in (1, 2):
        e, o = cl.handle(), cl.oracle()
        ref = o.schedule_batch(c_off, units.astype(np.int64))
        compare_outputs(ref, e.schedule_batch(c_off, units, mode=mode), f"mode {mode}")
        compare_rows(e, o, range(n_nodes))
        assert (ref["status"] == 3).sum() > 0 or n_nodes > 1000
