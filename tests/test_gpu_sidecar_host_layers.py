"""The drop-in layers with pods of 5..8 containers: the C++ twin of the plugin (csrc/host, `c_max` constructor
argument), its extender routes (egsr_*), and the C test double of the Go shim (integration/shim_double.c, `c_max` as
third command-line argument) run pods with sidecars on sidecar handles, and every answer, annotation, response body
and Status() row is checked against the C oracle.  With the default c_max every layer still refuses such pods."""
import json

import numpy as np
import pytest

import oracle_c as oc
from scenario import CBackend, make_scenario, run_scenario
from shim_double import ShimDoubleBackend, build_double

pytestmark = pytest.mark.gpu

CORE, MEM = "elasticgpu.io/gpu-core", "elasticgpu.io/gpu-memory"
SENT = (-1, -1, 0)


class SidecarShimDouble(ShimDoubleBackend):
    """The shim double started as `shim_double <policy> 8 <c_max>`."""

    def __init__(self, policy, c_max):
        import subprocess
        self.p = subprocess.Popen([build_double(), str(policy), "8", str(c_max)], stdin=subprocess.PIPE,
                                  stdout=subprocess.PIPE, text=True)
        self.n = 0
        self.g = {}


def _sidecar_shape(rng):
    """5..8 containers, at most 6 of them branching (fractional or no GPU request), the rest whole GPUs."""
    C = int(rng.integers(5, 9))
    out, nb = [], 0
    for _ in range(C):
        k = int(rng.integers(0, 3)) if nb < 6 else 1
        if k == 0:
            out.append((int(rng.choice([5, 10, 20, 30])), int(rng.integers(1, 6)), 0)); nb += 1
        elif k == 1:
            out.append((0, 0, 1))
        else:
            out.append(SENT); nb += 1
    return tuple(out)


def _sidecar_scenario(seed):
    rng = np.random.default_rng(seed)
    nodes, ops = make_scenario(seed, n_ops=30)
    shapes = [_sidecar_shape(rng) for _ in range(3)]
    for i in range(10):
        shape = shapes[int(rng.integers(len(shapes)))]
        at = int(rng.integers(0, len(ops) + 1))
        ops.insert(at, ("sched", shape, 5000 + i) if i % 4 else
                   ("add_pod", shape, 6000 + i, int(rng.integers(0, 4)), int(rng.integers(0, 1 << 30))))
    return nodes, ops


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", range(4))
def test_shim_double_with_sidecars_vs_oracle(seed, policy):
    nodes, ops = _sidecar_scenario(8100 + 2 * seed + policy)
    ref = run_scenario(CBackend(policy), nodes, ops, policy)
    b = SidecarShimDouble(policy, 8)
    try:
        got = run_scenario(b, nodes, ops, policy)
    finally:
        b.close()
    assert ref == got
    assert any(r[0] == "sched" and len(r) > 4 for r in ref)


def test_shim_double_default_c_max_refuses_five_containers():
    b = ShimDoubleBackend(0)
    try:
        assert b.add_node(800, 8 * 16) == 0
        assert b._ask("ASSUME 5 30 4 0 0 0 0 0 0 0 0 | n0")[1] == "error"
    finally:
        b.close()


def _units(reqs):
    return [oc.unit_from_requests(r.get("core", 0), r.get("memory", 0)) for r in reqs]


@pytest.mark.parametrize("policy", [0, 1])
def test_cpp_twin_with_sidecars_vs_oracle(policy):
    import egs_b200.host as H
    rng = np.random.default_rng(60 + policy)
    s = H.CudaUnitScheduler(policy, c_max=8)
    o = oc.OracleC(policy)
    names = []
    for i in range(8):
        g = int(rng.choice([1, 2, 4, 8, 8]))
        core, mem = 100 * g, g * int(rng.choice([16, 80]))
        names.append(f"n{i}")
        s.register_node(names[-1], core, mem)
        assert o.add_node(core, mem) == i
    placed = 0
    for k in range(60):
        nc = int(rng.integers(1, 9))
        reqs = [{"core": 100} if t == 0 else {} if t < 4 else {"core": int(rng.choice([10, 25, 50])), "memory": int(rng.integers(1, 8))}
                for t in (int(rng.integers(0, 8)) for _ in range(nc))]
        if not any(reqs) or sum(1 for r in reqs if r.get("core", 0) < 100) > 6:
            continue
        pod = H.Pod(f"p{k}", [(f"c{j}", r) for j, r in enumerate(reqs)])
        req = _units(reqs)
        filtered, failed, err = s.Assume(names, pod)
        assert err is None
        fit = o.filter(None, req)
        assert filtered == [n for n, f in zip(names, fit) if f] and set(failed) == {n for n, f in zip(names, fit) if not f}
        if not filtered:
            continue
        ids = [i for i in range(len(names)) if fit[i]]
        ost, sc = o.score(ids, req)
        assert ost == 0 and s.Score(filtered, pod) == [int(x) for x in sc]
        w = ids[int(np.argmax(sc))]
        st, alloc = o.bind(w, req, k)
        e = s.Bind(names[w], pod)
        assert (e is None) == (st == 0), e
        if st == 0:
            ann = s.pod_meta(pod)[0]
            assert [ann[f"elasticgpu.io/container-c{j}"] for j in range(nc)] == [",".join(map(str, a)) for a in alloc]
            placed += nc > 4
    status = json.loads(s.Status())
    for i, n in enumerate(names):
        assert [(g["CoreAvailable"], g["MemoryAvailable"]) for g in status[n]] == o.rows(i)
    assert placed > 0


def test_cpp_twin_default_c_max_refuses_five_containers():
    import egs_b200.host as H
    s = H.CudaUnitScheduler(0)
    s.register_node("a", 800, 8 * 16)
    pod = H.Pod("p", [("main", {"core": 30, "memory": 4})] + [(f"s{j}", {}) for j in range(4)])
    f, failed, err = s.Assume(["a"], pod)
    assert f == [] and "more than 4 containers" in err
    assert "more than 4 containers" in s.Bind("a", pod)
    wide = H.CudaUnitScheduler(0, c_max=8)
    wide.register_node("a", 800, 8 * 16)
    assert wide.Assume(["a"], pod)[0] == ["a"] and wide.Bind("a", pod) is None


def _go(obj) -> str:
    return json.dumps(obj, separators=(",", ":"))


def test_extender_routes_with_sidecars_vs_oracle():
    import egs_b200.host as H
    names = [f"node-{i:03d}" for i in range(40)]
    s = H.CudaUnitScheduler(0, max_nodes=64, c_max=8)
    o = oc.OracleC(0)
    for i, n in enumerate(names):
        core_alloc, mem_alloc = 100 * (1 + i % 8), 16 * (1 + i % 8)
        s.register_node(n, core_alloc, mem_alloc)
        o.add_node(core_alloc, mem_alloc)
    R = H.ExtenderRoutes(s)
    shapes = [[("main", {CORE: "30", MEM: "8"})] + [(f"side{j}", {}) for j in range(4)],             # 5 branching
              [("main", {CORE: "200"}), ("b", {CORE: "20", MEM: "1"})] + [(f"s{j}", {}) for j in range(5)],
              [("a", {CORE: "10", MEM: "2"}), ("b", {CORE: "10", MEM: "2"})] + [(f"s{j}", {}) for j in range(6)]]
    for k in range(12):
        cont = shapes[k % len(shapes)]
        req = [oc.unit_from_requests(int(r.get(CORE, 0)), int(r.get(MEM, 0))) for _, r in cont]
        pj = {"metadata": {"name": f"pod-{k}", "namespace": "default", "uid": f"uid-{k}"},
              "spec": {"containers": [{"name": n, "resources": {"requests": r, "limits": r}} for n, r in cont]},
              "status": {"phase": "Pending"}}
        fit = o.filter(None, req)
        filtered = [n for n, f in zip(names, fit) if f]
        want = {"nodenames": filtered}
        failed = {n: "no enough resource to allocate" for n, f in zip(names, fit) if not f}
        if failed:
            want["failedNodes"] = dict(sorted(failed.items()))
        st, got = R.filter(_go({"pod": pj, "nodes": None, "nodenames": names}).encode())
        assert st == 200 and got == _go(want), f"filter body differs at pod {k}"
        if not filtered:
            continue
        ost, sc = o.score([names.index(n) for n in filtered], req)
        st, got = R.priorities(_go({"pod": pj, "nodenames": filtered}).encode())
        assert st == 200 and got == _go([{"host": n, "score": int(x)} for n, x in zip(filtered, sc)])
        w = filtered[list(sc).index(max(sc))]
        pod = H.Pod(f"pod-{k}", [(n, {kk: int(v) for kk, v in (("core", r.get(CORE)), ("memory", r.get(MEM))) if v is not None})
                                 for n, r in cont], uid=f"uid-{k}")
        R.register_pod(pod)
        bst, _ = o.bind(names.index(w), req, k)
        st, got = R.bind(_go({"podName": f"pod-{k}", "podNamespace": "default", "podUID": f"uid-{k}", "node": w}).encode())
        assert (st, got) == (200, "{}") if bst == 0 else st == 500
    status = json.loads(s.Status())
    for i, n in enumerate(names):
        assert [(g["CoreAvailable"], g["MemoryAvailable"]) for g in status[n]] == o.rows(i)
