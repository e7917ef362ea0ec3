"""The indexed oracle driver (egso_schedule_batch_indexed) against the plain one (egso_schedule_batch), on the CPU.

The indexed driver re-Assumes only the nodes bound since a shape's last pod and keeps each shape's fit set in a max
index, which is what makes whole benchmark batches checkable.  Both drivers run the same operations on two oracle
objects; after every batch they must agree on the six per-pod outputs, the rows of every node, the cached option of
every shape on every node, and podMaps / releasedPodMap."""
import os
import subprocess
import sys
import time

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import oracle_c as oc

NPROC = os.cpu_count() or 1
ST_OK, ST_NOFIT, ST_TRANSACT = 0, 1, 3
# Two one-container requests whose GPURequest.Hash strings share the 8-hex sha256 prefix 269635e5.
FAITHFUL_TWINS = ((1, 15340, 0), (1, 35489, 0))


# ------------------------------------------------------------------------------------------------ generator
def random_nodes(rng, n, pressure):
    """[(G, mem per GPU, core row, mem row)]: 1 to 16 GPUs, each GPU full, partly used, empty or above its totals."""
    nodes = []
    for _ in range(n):
        G = int(rng.integers(1, 17))
        mt = int(rng.choice([1000, 4000, 16000]))
        kind = rng.choice(4, G, p=[0.15, 0.6, 0.15, 0.1] if pressure else [0.4, 0.35, 0.1, 0.15])
        core = np.where(kind == 0, 100, np.where(kind == 1, rng.integers(1, 100, G), np.where(kind == 2, 0, 100 + rng.integers(1, 50, G))))
        mem = np.where(kind == 0, mt, np.where(kind == 1, rng.integers(1, mt, G), np.where(kind == 2, 0, mt + rng.integers(1, 500, G))))
        nodes.append((G, mt, core.astype(np.int64), mem.astype(np.int64)))
    return nodes


def random_unit(rng, pressure):
    k = rng.choice(3, p=[0.2, 0.1, 0.7])
    if k == 0:
        return (0, 0, int(rng.integers(1, 5)))                       # whole GPUs
    if k == 1:
        return oc.unit_from_requests(0, 0)                            # the "no GPU needed" sentinel
    hi = 60 if pressure else 40
    return (int(rng.integers(1, hi)), int(rng.integers(1, 6000 if pressure else 3000)), 0)


def random_shapes(rng, n_shapes, pressure):
    """Trade tries every GPU for each fractional or sentinel container, G^C leaves on a G-GPU node: past 3 containers
    all but 2 of them take whole GPUs (the first free ones, no branching)."""
    shapes = []
    while len(shapes) < n_shapes:
        C = 1 if rng.random() < 0.6 else int(rng.integers(2, 9))      # 1, or 2 to 8 containers
        sh = [random_unit(rng, pressure) for _ in range(C)]
        if C > 3:
            for c in rng.permutation(C)[2:]:
                sh[c] = (0, 0, int(rng.integers(1, 3)))
        sh = tuple(sh)
        if sh not in shapes:
            shapes.append(sh)
    return shapes


def random_batch(rng, shapes, P):
    pick = rng.integers(0, len(shapes), P)
    reqs = [shapes[i] for i in pick]
    c_off = np.zeros(P + 1, np.int32)
    c_off[1:] = np.cumsum([len(r) for r in reqs])
    units = np.array([u for r in reqs for u in r], np.int64).reshape(-1, 3)
    return reqs, c_off, units


def mask_alloc(mask, req):
    return [[g for g in range(8) if (int(mask[c]) >> g) & 1] for c in range(len(req))]


def new_oracle(policy, nodes, faithful=False):
    o = oc.OracleC(policy, faithful)
    for n, (G, mt, core, mem) in enumerate(nodes):
        assert o.add_node(100 * G, mt * G) == n
        o.set_rows(n, core, mem)
    return o


# ------------------------------------------------------------------------------------------------ comparison
def assert_same_outputs(ref, got, what):
    d = oc.first_difference(ref, got)
    assert d is None, f"{what}: pod {d[0]}: {d[1]} differs (plain {ref[d[1]][d[0]]}, indexed {got[d[1]][d[0]]})"


def assert_same_state(a, b, n_nodes, shapes, uids):
    ids = np.arange(n_nodes)
    ra, rb = a.rows_many(ids, 16), b.rows_many(ids, 16)
    for x, y, name in zip(ra, rb, ("core", "mem", "GPU count")):
        bad = np.nonzero((x != y).reshape(n_nodes, -1).any(1))[0]
        assert bad.size == 0, f"{name} rows differ first on node {bad[0]}"
    for sh in shapes:
        pa, sa, ma = a.peek_many(ids, list(sh), 8)
        pb, sb, mb = b.peek_many(ids, list(sh), 8)
        bad = np.nonzero((pa != pb) | (sa != sb) | (ma != mb).any(1))[0]
        assert bad.size == 0, f"shape {sh}: cached option differs first on node {bad[0]}"
    for u in uids:
        assert a.known_pod(int(u)) == b.known_pod(int(u)), f"podMaps differs on uid {u}"
        assert a.released_pod(int(u)) == b.released_pod(int(u)), f"releasedPodMap differs on uid {u}"


def run_pair(seed, policy, n_nodes, n_shapes, pods, pressure=False, cache_load=False, muts=False, faithful=False):
    """The same operations on a plain-driver oracle and an indexed-driver oracle: an optional cache_load start, then
    one batch per entry of `pods`, the indexed side splitting each batch into two calls, with add_pod / forget_pod
    between batches.  Returns the plain driver's outputs of every batch."""
    rng = np.random.default_rng(seed)
    nodes = random_nodes(rng, n_nodes, pressure)
    shapes = random_shapes(rng, n_shapes, pressure)
    a, b = new_oracle(policy, nodes, faithful), new_oracle(policy, nodes, faithful)
    if cache_load:                                          # stale entries before the first pod
        for sh in [s for s in shapes if len(s) <= 4][:3]:
            valid = rng.random(n_nodes) < 0.5
            score = rng.integers(-300, 3000, n_nodes)
            am = np.zeros((n_nodes, 4), np.uint8)
            for n, (G, *_rest) in enumerate(nodes):
                for c in range(len(sh)):
                    am[n, c] = 1 << int(rng.integers(0, min(G, 8)))
            for o in (a, b):
                assert o.cache_load(list(sh), valid, score, am) == 0
    outs, all_uids, uid0 = [], [], 1
    for bi, P in enumerate(pods):
        reqs, c_off, units = random_batch(rng, shapes, P)
        uids = np.arange(uid0, uid0 + P, dtype=np.uint64)
        if bi % 2:                                          # repeated uids: a bind onto a node whose podsMap holds it
            uids = uids[rng.integers(0, max(1, P // 2), P)]
        uid0 += P
        all_uids.extend(int(u) for u in uids)
        ref = a.schedule_batch(c_off, units, uids, threads=2)
        k = int(rng.integers(0, P + 1))
        got0 = b.schedule_batch_indexed(c_off[:k + 1], units[:int(c_off[k])], uids[:k], threads=2)
        got1 = b.schedule_batch_indexed(c_off[k:] - c_off[k], units[int(c_off[k]):], uids[k:], threads=1)
        got = {f: np.concatenate([got0[f], got1[f]]) for f in oc.FIELDS}
        assert_same_outputs(ref, got, f"seed {seed}, batch {bi} (split at {k})")
        assert_same_state(a, b, n_nodes, shapes, all_uids)
        outs.append(ref)
        if muts:
            bound = np.nonzero((ref["status"] == ST_OK) & (np.diff(c_off) <= 4))[0]
            for p in rng.choice(bound, min(len(bound), 8), replace=False) if len(bound) else []:
                rec = (int(ref["node"][p]), list(reqs[p]), mask_alloc(ref["alloc_mask"][p], reqs[p]), int(uids[p]))
                for o in (a, b):
                    o.forget_pod(*rec)
            for _ in range(6):
                n = int(rng.integers(0, n_nodes))
                sh = shapes[int(rng.integers(0, len(shapes)))]
                alloc = [sorted(rng.choice(nodes[n][0], min(u[2] or 1, nodes[n][0]), replace=False).tolist()) for u in sh]
                all_uids.append(uid0)
                for o in (a, b):
                    o.add_pod(n, list(sh), alloc, uid0)
                uid0 += 1
            for o in (a, b):
                o.forget_pod(-1, [(1, 1, 0)], [[0]], 10 ** 9)
            assert_same_state(a, b, n_nodes, shapes, all_uids)
    return outs


# ------------------------------------------------------------------------------------------------ random clusters
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", range(4))
def test_random_clusters(policy, seed):
    run_pair(seed, policy, n_nodes=60, n_shapes=10, pods=[300])


@pytest.mark.parametrize("policy", [0, 1])
def test_pressure_nofit_and_transact(policy):
    """A small, mostly used cluster under many pods: both Filter finding nothing and a stale cached option failing
    its Transact happen, and the drivers agree through them."""
    outs = run_pair(11, policy, n_nodes=12, n_shapes=8, pods=[400], pressure=True)
    status = outs[0]["status"]
    assert (status == ST_NOFIT).any() and (status == ST_TRANSACT).any(), np.bincount(status)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", range(3))
def test_batches_compose_with_verbs_between(policy, seed):
    """Several batches on one object, a cache_load start (stale entries before the first pod), add_pod / forget_pod
    between batches, and each indexed batch split into two calls."""
    run_pair(100 + seed, policy, n_nodes=40, n_shapes=8, pods=[150, 200, 120], pressure=seed == 2,
             cache_load=True, muts=True)


def test_faithful_mode_agrees_with_distinct_keys():
    run_pair(7, 0, n_nodes=30, n_shapes=6, pods=[200, 100], faithful=True, muts=True)


def test_faithful_mode_refuses_a_shared_key():
    assert oc.request_hash([FAITHFUL_TWINS[0]]) == oc.request_hash([FAITHFUL_TWINS[1]])
    o = new_oracle(0, [(2, 40000, np.array([100, 100]), np.array([40000, 40000]))], faithful=True)
    units = np.array(FAITHFUL_TWINS, np.int64)
    with pytest.raises(ValueError):
        o.schedule_batch_indexed(np.array([0, 1, 2], np.int32), units)
    assert o.rows(0) == [(100, 40000), (100, 40000)] and not o.known_pod(0)


@settings(max_examples=80, deadline=None)
@given(seed=st.integers(0, 2 ** 32 - 1), policy=st.integers(0, 1), n_nodes=st.integers(1, 40),
       n_shapes=st.integers(1, 8), pods=st.lists(st.integers(0, 120), min_size=1, max_size=3),
       pressure=st.booleans(), cache_load=st.booleans(), muts=st.booleans())
def test_property(seed, policy, n_nodes, n_shapes, pods, pressure, cache_load, muts):
    run_pair(seed, policy, n_nodes, n_shapes, pods, pressure, cache_load, muts)


# ------------------------------------------------------------------------------------------------ benchmark configs
def workload(cfg, n_pods=None):
    import egs_b200
    return egs_b200.workloads.config(cfg, n_pods=n_pods)


def workload_oracle(w):
    o = oc.OracleC(w.policy)
    assert o.add_nodes(w.gpus, w.mem_total * w.gpus, w.core, w.mem) == 0
    return o


@pytest.mark.parametrize("cfg,n_pods", [(1, None), (2, None), (4, 1000), (3, 400)])
def test_benchmark_config_equals_plain_driver(cfg, n_pods):
    """Configs 1 and 2 whole; configs 4 and 3 (all their nodes) on a pod prefix the plain driver can afford."""
    w = workload(cfg, n_pods)
    a, b = workload_oracle(w), workload_oracle(w)
    ref = a.schedule_batch(w.c_off, w.units64(), threads=NPROC)
    got = b.schedule_batch_indexed(w.c_off, w.units64(), threads=NPROC)
    assert_same_outputs(ref, got, f"cfg{cfg}")
    ids = np.arange(w.n_nodes)
    for x, y in zip(a.rows_many(ids, 8), b.rows_many(ids, 8)):
        assert np.array_equal(x, y), f"cfg{cfg}: rows differ"
    import egs_b200
    for sh in egs_b200.workloads.shapes_of(w):
        for x, y in zip(a.peek_many(ids, list(sh)), b.peek_many(ids, list(sh))):
            assert np.array_equal(x, y), f"cfg{cfg}: cached options of {sh} differ"


@pytest.mark.parametrize("cfg", [4, 3])
def test_full_size_wall_time(cfg, capsys):
    """The indexed driver on a whole benchmark batch; prints its wall time."""
    w = workload(cfg)
    o = workload_oracle(w)
    t0 = time.perf_counter()
    out = o.schedule_batch_indexed(w.c_off, w.units64(), threads=NPROC)
    dt = time.perf_counter() - t0
    with capsys.disabled():
        print(f"\nindexed oracle, cfg{cfg} ({w.n_nodes} nodes, {w.n_pods} pods, {NPROC} threads): {dt:.1f} s")
    assert ((out["node"] >= 0) == (out["status"] != ST_NOFIT)).all()
    assert (out["fit_count"][out["node"] >= 0] > 0).all()


# ------------------------------------------------------------------------------------------------ the helpers
@pytest.mark.parametrize("faithful", [False, True])
def test_peek_many_equals_peek_on_each_node(faithful):
    """The bulk cache read the state comparisons use against the one-node verb, on 1- to 16-GPU nodes and 1 to 8
    containers."""
    rng = np.random.default_rng(5)
    nodes = random_nodes(rng, 50, False)
    shapes = random_shapes(rng, 10, False)
    o = new_oracle(1, nodes, faithful)
    _reqs, c_off, units = random_batch(rng, shapes, 200)
    o.schedule_batch_indexed(c_off, units)
    n_present = 0
    for sh in shapes:
        present, score, masks = o.peek_many(range(len(nodes)), list(sh), 8)
        for n in range(len(nodes)):
            one = o.peek(n, list(sh))
            assert present[n] == (one is not None), (sh, n)
            if one is not None:
                n_present += 1
                assert score[n] == one[1] and masks[n, :len(sh)].tolist() == [sum(1 << g for g in a) for a in one[0]]
                assert not masks[n, len(sh):].any()
    assert n_present > 0


def test_first_difference_names_pod_and_field():
    w = workload(1, 500)
    ref = workload_oracle(w).schedule_batch_indexed(w.c_off, w.units64())
    assert oc.first_difference(ref, {f: ref[f].copy() for f in oc.FIELDS}) is None
    for f, p in (("score_digest", 321), ("alloc_mask", 17), ("node", 499), ("status", 0)):
        got = {g: ref[g].copy() for g in oc.FIELDS}
        got[f][p] ^= 1
        got["fit_count"][p + 1:] += 1                       # later differences do not hide the first
        assert oc.first_difference(ref, got) == (p, f)
        with pytest.raises(AssertionError, match=f"pod {p}: {f} differs"):
            assert_same_outputs(ref, got, "perturbed")


def test_verify_bench_dump_tool(tmp_path):
    """tools/verify_bench_dump.py on a dump written by bench.py's own dump_outputs: exit 0 on the oracle's answer,
    1 naming the first differing pod and field on a perturbed one."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import importlib
    bench = importlib.import_module("bench")
    w = workload(1)
    ref = workload_oracle(w).schedule_batch_indexed(w.c_off, w.units64())
    tool = [sys.executable, os.path.join(root, "tools", "verify_bench_dump.py"), str(tmp_path), "--cfg", "1"]
    bench.dump_outputs(str(tmp_path), ref)
    r = subprocess.run(tool, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    bad = {f: ref[f].copy() for f in oc.FIELDS}
    bad["fit_digest"][4321] += np.uint64(1 << 40)           # only the high half changes
    bad["node"][9000] += 1
    bench.dump_outputs(str(tmp_path), bad)
    r = subprocess.run(tool, capture_output=True, text=True, timeout=600)
    assert r.returncode == 1 and "pod 4321: fit_digest differs" in r.stdout, r.stdout + r.stderr
