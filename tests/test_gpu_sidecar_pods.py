"""Sidecar handles (egs_create_ex with c_max > 4): pods of 5..8 containers through filter, score, bind, peek,
option_dump and the per-pod batch engine, against the C oracle, on both sides of the one-thread DFS / leaf-split
threshold.  The oracle's own verbs are driven pod by pod (oracle_batch with 8 planes), so that all 8 masks of a pod
are compared."""
import ctypes as C

import numpy as np
import pytest

from oracle_harness import FIELDS, Cluster, compare_caches, compare_outputs, compare_rows, egs, oracle_batch

pytestmark = pytest.mark.gpu

SENT = (-1, -1, 0)


def _pair(policy, nodes, g_max=8):
    """nodes: [(gpus, mem_total, rows or None)] on a sidecar handle and on the oracle."""
    cl = Cluster(policy, nodes, g_max, c_max=8)
    return cl.handle(), cl.oracle()


def _batch(pods):
    c_off = np.cumsum([0] + [len(p) for p in pods]).astype(np.int32)
    units = np.array([u for p in pods for u in p], np.int32).reshape(-1, 3)
    return c_off, units


def _cluster(rng, n):
    nodes = []
    for _ in range(n):
        g = int(rng.integers(1, 9))
        mt = 32
        core = [int(rng.choice([100, 100, 100, 60, 0, 37])) for _ in range(g)]
        mem = [mt if c == 100 else int(rng.integers(0, mt + 1)) for c in core]
        nodes.append((g, mt, (core, mem)))
    return nodes


def _pod(rng, n_branch_max=5):
    """5..8 containers: one or two GPU containers, whole-GPU ones and sentinels (at most n_branch_max branching)."""
    C_ = int(rng.integers(5, 9))
    out, nb = [], 0
    for _ in range(C_):
        k = int(rng.integers(0, 3))
        if nb >= n_branch_max:
            k = 1
        if k == 0:
            out.append((int(rng.integers(5, 60)), int(rng.integers(1, 12)), 0)); nb += 1
        elif k == 1:
            out.append((0, 0, int(rng.integers(1, 3))))
        else:
            out.append(SENT); nb += 1
    return out


# ------------------------------------------------------------------------------------------------ refusals
def test_create_ex_arguments():
    cap = egs().capi
    L = cap.load()
    h = C.c_void_p()
    for g, c in ((8, 0), (8, 9), (16, 5), (9, 8)):
        assert L.egs_create_ex(0, 16, g, c, 0, C.byref(h)) == cap.EGS_ERR_BAD_ARG
    for g, c in ((8, 1), (16, 4), (8, 5), (4, 8)):
        assert L.egs_create_ex(0, 16, g, c, 0, C.byref(h)) == cap.EGS_OK
        L.egs_destroy(h)


def test_sidecar_limits_are_refused_with_a_text():
    cap = egs().capi
    e, o = _pair(0, [(8, 32, None)] * 4)
    pods = [[(10, 4, 0)] + [SENT] * 4]
    c_off, units = _batch(pods)
    with pytest.raises(cap.EgsError, match="c_max"):
        e.schedule_batch(c_off, units, mode=cap.EGS_MODE_ROUNDS)
    rec = [(cap.EGS_MUT_ADD, 0, [(30, 8, 0)], [[0]], 77)]
    with pytest.raises(cap.EgsError, match="c_max"):
        e.schedule_batch_mut(c_off, units, [0], rec, mode=cap.EGS_MODE_ROUNDS)
    assert e.rows(0)[0] == (100, 32) and not e.pod_known(77)           # the record was not applied
    with pytest.raises(cap.EgsError, match="c_max"):
        e.shard_set(0, 2)
    with pytest.raises(cap.EgsError, match="EGS_MAX_CONTAINERS"):
        e.profile_evaluate(pods[0], iters=1)
    with pytest.raises(cap.EgsError):
        e.filter(None, [SENT] * 9)
    d = egs().Egs(0, 4, 8)                                                 # a default handle still refuses 5
    with pytest.raises(cap.EgsError):
        d.filter(None, pods[0])


def test_device_masks_need_8_byte_alignment():
    cap = egs().capi
    import torch
    e, o = _pair(0, [(8, 32, None)] * 4)
    c_off, units = _batch([[(10, 4, 0)] + [SENT] * 4] * 2)
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    with pytest.raises(cap.EgsError, match="aligned"):
        e.schedule_batch_device(c_off, units, [0, 0, buf.data_ptr() + 4, 0, 0, 0])
    e.schedule_batch_device(c_off, units, [0, 0, buf.data_ptr() + 8, 0, 0, 0])
    torch.cuda.synchronize()
    ref = oracle_batch(o, c_off, units, np.arange(2) + 1000000, planes=8)
    assert np.array_equal(buf[8:24].cpu().numpy().reshape(2, 8), ref["alloc_mask"])


# ------------------------------------------------------------------------------------------------ hand cases
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("n_sent", [4, 5, 8])
def test_last_maximal_leaf_under_ties(policy, n_sent):
    """Equal GPUs: every leaf ties and the last one wins -- on both sides of the threshold (4 sentinels: DFS)."""
    e, o = _pair(policy, [(8, 32, None), (5, 32, None)])
    req = [SENT] * n_sent + [(0, 0, 1)] * (5 - n_sent if n_sent < 5 else 0)
    assert list(e.filter(None, req)) == list(o.filter(None, req))
    for i in range(2):
        assert e.peek(i, req) == o.peek(i, req)
    compare_caches(e, o, [req], range(2), unfit_check=True)


def test_sentinel_makes_a_whole_gpu_container_skip_a_gpu():
    rows = ([100, 100, 40, 100, 100, 100, 100, 100], [32, 32, 8, 32, 32, 32, 32, 32])
    e, o = _pair(0, [(8, 32, rows)])
    req = [SENT, SENT, (0, 0, 2), SENT, SENT, (0, 0, 1), SENT]     # 5 branching: the leaf-split kernels
    assert list(e.filter(None, req)) == list(o.filter(None, req)) == [1]
    assert e.peek(0, req) == o.peek(0, req)
    assert e.bind(0, req, 5) == o.bind(0, req, 5)
    compare_rows(e, o, range(1))


def test_stale_option_fails_in_transact():
    e, o = _pair(0, [(8, 32, None), (4, 32, None)])
    req = [(0, 0, 2)] + [SENT] * 5
    assert list(e.filter(None, req)) == list(o.filter(None, req))
    other, alloc = [(0, 0, 1)], [[1]]                        # GPU 1 of the cached option is taken meanwhile
    assert e.pod_apply(0, other, alloc, 9) == 0 and o.add_pod(0, other, alloc, 9) == 0
    got = e.bind(0, req, 10)
    assert got == o.bind(0, req, 10) and got[0] == egs().capi.EGS_ERR_TRANSACT
    compare_rows(e, o, range(2))
    compare_caches(e, o, [req], range(2), unfit_check=True)


@pytest.mark.parametrize("policy", [0, 1])
def test_two_bit_digits_on_a_four_gpu_sidecar_handle(policy):
    """g_max = 4: digits are 2 bits wide, so 7 branching containers (2^14 leaves) take the leaf-split kernels, and a
    node with fewer GPUs meets digits that name absent GPUs."""
    rows = ([100, 37, 100], [32, 9, 32])
    e, o = _pair(policy, [(4, 32, None), (3, 32, rows), (1, 32, None), (2, 32, ([60, 0], [20, 0]))], 4)
    for req in ([(10, 4, 0)] + [SENT] * 6, [SENT, (0, 0, 1), SENT, (20, 5, 0)] + [SENT] * 4, [SENT] * 6):
        assert list(e.filter(None, req)) == list(o.filter(None, req)), req
        compare_caches(e, o, [req], range(4), unfit_check=True)
        for i in range(4):
            assert e.bind(i, req, 40 + i) == o.bind(i, req, 40 + i)
        compare_rows(e, o, range(4))


@pytest.mark.parametrize("req", [[SENT] * 5, [SENT] * 4 + [(0, 0, 1)]])
def test_score_without_filter_is_the_reference_panic(req):
    rows = ([0] * 6 + [100, 100], [0] * 6 + [32, 32])
    e, o = _pair(0, [(8, 32, rows), (8, 32, None), (3, 32, None)])
    e.filter([1], req); o.filter([1], req)
    st, sc = e.score([0, 1, 2], req)
    ost, osc = o.score([0, 1, 2], req)
    assert st == ost == egs().capi.EGS_ERR_PANIC and list(sc) == list(osc)
    compare_caches(e, o, [req], range(3), unfit_check=True)


@pytest.mark.parametrize("policy", [0, 1])
def test_one_node_with_2_24_leaves(policy):
    """Eight branching containers on one 8-GPU node: the whole leaf space goes over the grid."""
    rows = ([101, 0, 37, 100, 99, 1, 100, 60], [41, 0, 9, 32, 31, 1, 32, 2])
    e, o = _pair(policy, [(8, 32, rows)])
    req = [(30, 8, 0), SENT, (20, 20, 0)] + [SENT] * 5
    assert list(e.filter(None, req)) == list(o.filter(None, req)) == [1]
    assert e.peek(0, req) == o.peek(0, req)
    assert e.bind(0, req, 1) == o.bind(0, req, 1)
    compare_rows(e, o, range(1))


# ------------------------------------------------------------------------------------------------ sequences
@pytest.mark.parametrize("policy,seed", [(0, 1), (1, 2), (0, 3)])
def test_verb_sequences_against_the_oracle(policy, seed):
    rng = np.random.default_rng(seed)
    n = 24
    e, o = _pair(policy, _cluster(rng, n))
    shapes = [tuple(_pod(rng, 5 if k % 2 else 3)) for k in range(5)] + [((10, 4, 0),), ((0, 0, 1), SENT)]
    uid = 100
    for step in range(40):
        sh = list(shapes[int(rng.integers(0, len(shapes)))])
        ids = rng.choice(n, int(rng.integers(1, n + 1)), replace=False).astype(np.int32)   # an extender's node list
        verb = int(rng.integers(0, 4))
        if verb == 0:
            assert list(e.filter(ids, sh)) == list(o.filter(ids, sh)), f"step {step} filter"
        elif verb == 1:
            st, sc = e.score(ids, sh)
            ost, osc = o.score(ids, sh)
            assert st == ost and list(sc) == list(osc), f"step {step} score"
        elif verb == 2:
            w = int(ids[0]); uid += 1
            assert e.bind(w, sh, uid) == o.bind(w, sh, uid), f"step {step} bind"
        else:
            w = int(rng.integers(0, n)); uid += 1
            g = o.gpu_count(w)
            rec = [(5, 2, 0), (0, 0, 1)]
            alloc = [[int(rng.integers(0, g))], [int(rng.integers(0, g))]]
            assert e.pod_apply(w, rec, alloc, uid) == o.add_pod(w, rec, alloc, uid)
        compare_rows(e, o, range(n))
        compare_caches(e, o, shapes, range(n), unfit_check=True)


@pytest.mark.parametrize("policy", [0, 1])
def test_batches_against_the_oracle_driver(policy):
    cap = egs().capi
    rng = np.random.default_rng(7 + policy)
    nodes = _cluster(rng, 40)
    pods = [_pod(rng, 5 if p % 3 else 3) for p in range(30)] + [[(10, 4, 0)], [(0, 0, 2), SENT]]
    c_off, units = _batch(pods)
    ref = oracle_batch(Cluster(policy, nodes).oracle(), c_off, units, np.arange(len(pods)) + 1000000, planes=8)
    for call in ("batch", "mut", "vec", "device"):
        e, o = _pair(policy, nodes)
        if call == "batch":
            got = e.schedule_batch(c_off, units)
        elif call == "mut":
            got = e.schedule_batch_mut(c_off, units, [], [], mode=cap.EGS_MODE_RESCAN)
        elif call == "vec":
            got = e.schedule_batch_vec(c_off, units, 3)
        else:
            import torch
            P = len(pods)
            t = dict(node=torch.zeros(P, dtype=torch.int32, device="cuda"), status=torch.zeros(P, dtype=torch.int32, device="cuda"),
                     alloc_mask=torch.zeros(P * 8, dtype=torch.uint8, device="cuda"), fit_count=torch.zeros(P, dtype=torch.int32, device="cuda"),
                     fit_digest=torch.zeros(P, dtype=torch.int64, device="cuda"), score_digest=torch.zeros(P, dtype=torch.int64, device="cuda"))
            e.schedule_batch_device(c_off, units, [t[f].data_ptr() for f in FIELDS])
            torch.cuda.synchronize()
            got = {f: t[f].cpu().numpy() for f in FIELDS}
            got["alloc_mask"] = got["alloc_mask"].reshape(P, 8)
            got["fit_digest"] = got["fit_digest"].view(np.uint64); got["score_digest"] = got["score_digest"].view(np.uint64)
        compare_outputs(ref, got, call)
        if call == "batch":
            oracle_batch(o, c_off, units, np.arange(len(pods)) + 1000000, planes=8)
            compare_rows(e, o, range(len(nodes)))
            compare_caches(e, o, [tuple(p) for p in pods[:6]], range(len(nodes)), unfit_check=True)


def test_oracle_driver_equals_egso_schedule_batch():
    """Pins the harness driver's 8-plane mode to the oracle's own batch on pods of up to 4 containers."""
    rng = np.random.default_rng(11)
    nodes = _cluster(rng, 30)
    pods = [[(int(rng.integers(5, 60)), int(rng.integers(1, 12)), 0)] + [SENT] * int(rng.integers(0, 3)) for _ in range(25)]
    c_off, units = _batch(pods)
    uids = np.arange(len(pods), dtype=np.uint64) + 5
    a = oracle_batch(Cluster(0, nodes).oracle(), c_off, units, uids, planes=8)
    b = Cluster(0, nodes).oracle().schedule_batch(c_off, units.astype(np.int64), uids)
    for f in FIELDS:
        x = a[f][:, :4] if f == "alloc_mask" else a[f]
        assert np.array_equal(x, b[f]), f


def test_checkpoint_rollback_with_8_plane_tables():
    rng = np.random.default_rng(5)
    nodes = _cluster(rng, 20)
    e, o = _pair(0, nodes)
    pods = [_pod(rng, 5) for _ in range(10)]
    e.schedule_batch(*_batch(pods[:4]))
    shapes = [tuple(p) for p in pods]
    before = [e.option_dump(list(sh)) for sh in shapes[:4]]
    rows = e.state_dump()
    e.checkpoint_save()
    a = e.schedule_batch(*_batch(pods[4:]))
    e.checkpoint_rollback()
    for sh, (st, sc, am) in zip(shapes[:4], before):
        st2, sc2, am2 = e.option_dump(list(sh))
        assert np.array_equal(st, st2) and np.array_equal(sc[st == 1], sc2[st == 1]) and np.array_equal(am[st == 1], am2[st == 1])
    assert all(np.array_equal(x, y) for x, y in zip(rows, e.state_dump()))
    b = e.schedule_batch(*_batch(pods[4:]))
    compare_outputs(a, b, "after rollback")


@pytest.mark.parametrize("mode", [1, 2])
def test_small_pods_on_a_sidecar_handle_equal_a_default_handle(mode):
    cap = egs().capi
    w = egs().workloads.config(1, n_nodes=2000, n_pods=3000, policy=0)
    d = egs().Egs(w.policy, w.n_nodes, 8)
    s = egs().Egs(w.policy, w.n_nodes, 8, c_max=8)
    for x in (d, s):
        x.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
    a = d.schedule_batch(w.c_off, w.units, mode=mode)
    b = s.schedule_batch(w.c_off, w.units)
    for f in FIELDS:
        if f == "alloc_mask":
            assert np.array_equal(a[f], b[f][:, :4]) and not b[f][:, 4:].any()
        else:
            assert np.array_equal(a[f], b[f]), f
