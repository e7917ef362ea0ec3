"""The drop-in layers on servers with 10 and 16 GPUs: the C++ twin of the plugin (csrc/host, `g_max` constructor
argument) and the C test double of the Go shim (integration/shim_double.c, `g_max` command-line argument) run
scenarios with 9..16-GPU nodes and whole-GPU requests above 8, and every answer, annotation, mask and Status() row
is checked against the oracles."""
import json

import numpy as np
import pytest

import egs_oracle as po
from scenario import CBackend, make_scenario, run_scenario
from shim_double import ShimDoubleBackend

pytestmark = pytest.mark.gpu


def _wide_scenario(seed):
    """make_scenario's verbs on nodes of 9..16 GPUs (and a few narrow ones), plus whole-GPU pods of 9..16 GPUs."""
    rng = np.random.default_rng(seed)
    _, ops = make_scenario(seed, n_ops=50)
    nodes = []
    for _ in range(int(rng.integers(2, 6))):
        G = int(rng.choice([2, 8, 9, 10, 12, 16, 16]))
        M = int(rng.choice([12, 16, 80]))
        rows = None
        if rng.integers(0, 2):
            rows = ([int(rng.choice([100, 100, 100, 75, 50, 0])) for _ in range(G)],
                    [int(rng.integers(0, M + 1)) if rng.integers(0, 3) == 0 else M for _ in range(G)])
            rows = (rows[0], [M if c == 100 else m for c, m in zip(*rows)])
        nodes.append((G * 100 + int(rng.integers(0, 100)), G * M + int(rng.integers(0, G)), rows))
    big = [((0, 0, 12),), ((0, 0, 9),), ((0, 0, 16),), ((0, 0, 10), (5, 1, 0)), ((-1, -1, 0), (0, 0, 11))]
    for i in range(12):
        shape = big[int(rng.integers(len(big)))]
        at = int(rng.integers(0, len(ops) + 1))
        ops.insert(at, ("sched", shape, 3000 + i) if i % 3 else ("add_pod", shape, 4000 + i, int(rng.integers(0, 8)),
                                                                  int(rng.integers(0, 1 << 30))))
    return nodes, ops


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", range(6))
def test_shim_double_on_wide_nodes_vs_oracle(seed, policy):
    nodes, ops = _wide_scenario(7000 + 2 * seed + policy)
    ref = run_scenario(CBackend(policy), nodes, ops, policy)
    b = ShimDoubleBackend(policy, g_max=16)
    try:
        got = run_scenario(b, nodes, ops, policy)
    finally:
        b.close()
    assert ref == got
    assert any(len(r) for r in ref if r[0] == "rows")


def test_shim_double_default_width_refuses_a_ten_gpu_node():
    b = ShimDoubleBackend(0)
    try:
        assert b.add_node(1000, 10 * 16) == -1                    # g_max defaults to EGS_MAX_GPUS
        assert b.add_node(800, 8 * 16) == 0
    finally:
        b.close()


@pytest.mark.parametrize("policy", [0, 1])
def test_cpp_twin_on_wide_nodes_vs_oracle(policy):
    import egs_b200.host as H
    rng = np.random.default_rng(50 + policy)
    s = H.CudaUnitScheduler(policy, g_max=16)
    o = po.Scheduler(policy)
    names = []
    for i in range(10):
        g = int(rng.choice([10, 16, 12, 9, 2]))
        core, mem = 100 * g + int(rng.integers(0, 99)), g * int(rng.choice([16, 80]))
        names.append(f"n{i}")
        s.register_node(names[-1], core, mem)
        assert o.add_node(core, mem) == i
    big = 0
    for k in range(250):
        nc = int(rng.integers(1, 4))
        reqs = []
        for _ in range(nc):
            t = rng.integers(0, 10)
            reqs.append({} if t == 0 else {"core": 100 * int(rng.choice([1, 2, 9, 12, 16]))} if t == 1 else
                        {"core": int(rng.choice([0, 10, 25, 50])), "memory": int(rng.integers(0, 12))})
        if not any(reqs):
            continue
        pod = H.Pod(f"p{k}", [(f"c{j}", r) for j, r in enumerate(reqs)])
        req = po.new_gpu_request([(r.get("core", 0), r.get("memory", 0)) for r in reqs])
        filtered, failed, err = s.Assume(names, pod)
        assert err is None
        fit = o.assume(range(len(names)), req)
        assert filtered == [n for n, f in zip(names, fit) if f] and set(failed) == {n for n, f in zip(names, fit) if not f}
        if not filtered:
            continue
        ids = [i for i in range(len(names)) if fit[i]]
        sc = o.score(ids, req)
        assert s.Score(filtered, pod) == sc
        w = ids[sc.index(max(sc))]
        st, alloc = o.bind(w, req, k)
        e = s.Bind(names[w], pod)
        assert (e is None) == (st == 0), e
        if st == 0:
            ann = s.pod_meta(pod)[0]
            assert [ann[f"elasticgpu.io/container-c{j}"] for j in range(nc)] == [",".join(map(str, a)) for a in alloc]
            big += any(g >= 8 for a in alloc for g in a)
    status = json.loads(s.Status())
    for i, n in enumerate(names):
        assert [(g["CoreAvailable"], g["MemoryAvailable"]) for g in status[n]] == o.rows(i)
    assert big > 0 and max(len(status[n]) for n in names) == 16


def test_cpp_twin_whole_gpus_of_a_sixteen_gpu_server():
    import egs_b200.host as H
    s = H.CudaUnitScheduler(0, g_max=16)
    s.register_node("big", 1600, 16 * 80)
    pod = H.Pod("p", [("a", {"core": 1200}), ("b", {"core": 30, "memory": 8})])
    assert s.Assume(["big"], pod)[0] == ["big"]
    assert s.Bind("big", pod) is None
    ann = s.pod_meta(pod)[0]
    assert ann["elasticgpu.io/container-a"] == ",".join(map(str, range(12)))
    assert ann["elasticgpu.io/container-b"] == "15"              # binpack: the last maximal GPU (gpu.go:85)
    rows = json.loads(s.Status())["big"]
    assert len(rows) == 16 and rows[15]["CoreAvailable"] == 70 and rows[11]["CoreAvailable"] == 0
    narrow = H.CudaUnitScheduler(0)                               # g_max defaults to EGS_MAX_GPUS
    narrow.register_node("big", 1600, 16 * 80)
    f, failed, err = narrow.Assume(["big"], pod)
    assert f == [] and "get node failed" in failed["big"]
