"""Nodes of up to 16 GPUs on a wide handle (g_max > 8: 16-wide rows, u16 masks, the per-pod engine) against the C
oracle, which holds 16 GPUs per node: hand cases, seeded verb sequences on mixed clusters with every answer, row and
option cache checked after every step, the four batch calls, the guards of a wide handle, and the per-pod engine on a
wide handle against the rounds engine on an 8-wide one."""
import numpy as np
import pytest

import oracle_c as oc

pytestmark = pytest.mark.gpu

FIELDS = ["node", "status", "alloc_mask", "fit_count", "fit_digest", "score_digest"]
GS = [1, 2, 8, 9, 10, 12, 16]
M64 = (1 << 64) - 1
SHAPES = [
    [(10, 4, 0)], [(50, 8, 0)], [(25, 2, 0)], [(0, 6, 0)], [(-1, -1, 0)],
    [(0, 0, 1)], [(0, 0, 2)], [(0, 0, 9)], [(0, 0, 12)], [(0, 0, 16)],
    [(30, 2, 0), (0, 0, 2)], [(20, 4, 0), (-1, -1, 0), (10, 1, 0)], [(0, 0, 10), (5, 1, 0)],
    [(40, 3, 0), (40, 3, 0), (0, 0, 1), (-1, -1, 0)],
]


def _eg():
    import egs_b200
    return egs_b200


def _req(units, c_off, p):
    return [tuple(int(x) for x in units[k]) for k in range(int(c_off[p]), int(c_off[p + 1]))]


def _cluster(policy, n, seed, gs=GS):
    """A wide handle and the oracle over the same n nodes of G in `gs` GPUs, about half of them partly used."""
    eg = _eg()
    rng = np.random.default_rng(seed)
    e = eg.Egs(policy, n, 16)
    o = oc.OracleC(policy)
    for i in range(n):
        G = int(rng.choice(gs)); M = int(rng.choice([16, 32]))
        assert e.node_set_allocatable(i, 100 * G, M * G) == 0
        assert o.add_node(100 * G, M * G) == i
        if rng.integers(0, 2):
            core = [100 if rng.integers(0, 3) == 0 else int(rng.integers(0, 101)) for _ in range(G)]
            mem = [M if c == 100 else int(rng.integers(0, M + 1)) for c in core]
            assert e.state_load(i, core, mem) == 0
            o.set_rows(i, core, mem)
    return e, o, rng


def _check_rows(e, o, n):
    core, mem, gc, _ = e.state_dump()
    assert core.shape == (n, 16)
    for i in range(n):
        g = int(gc[i])
        assert [(int(core[i, k]), int(mem[i, k])) for k in range(g)] == o.rows(i), i
        assert (core[i, g:] == -(1 << 31)).all() and (mem[i, g:] == -(1 << 31)).all()


def _check_caches(e, o, n, shapes, rng):
    """option_dump of every shape on every node against the oracle's cache, and peek on a few nodes."""
    cap = _eg().capi
    for req in shapes:
        st, sc, am = e.option_dump(req)
        assert am.dtype == np.uint16
        for i in range(n):
            want = o.peek(i, req)
            if st[i] == 1:
                assert want == (cap.masks_to_lists(am[i], len(req)), int(sc[i])), (i, req)
            else:
                assert want is None, (i, req, st[i])
        for i in rng.choice(n, size=3, replace=False):
            assert e.peek(int(i), req) == o.peek(int(i), req)


def _oracle_batch(o, n, c_off, units, uids, muts=(), mut_at=()):
    """The driver rule on the oracle pod by pod with its own verbs -- filter every node, score the fit ones, bind the
    first maximal -- so the masks keep all 16 GPUs.  Records muts[j] apply right before pod mut_at[j]."""
    mix = o.L.egso_mix64
    P = len(c_off) - 1
    out = dict(node=np.full(P, -1, np.int32), status=np.zeros(P, np.int32), alloc_mask=np.zeros((P, 4), np.uint16),
               fit_count=np.zeros(P, np.int32), fit_digest=np.zeros(P, np.uint64), score_digest=np.zeros(P, np.uint64))
    j = 0
    for p in range(P):
        while j < len(mut_at) and mut_at[j] == p:
            _oracle_mut(o, muts[j]); j += 1
        req = _req(units, c_off, p)
        ids = np.flatnonzero(o.filter(None, req)).astype(np.int32)
        out["fit_count"][p] = len(ids)
        if len(ids) == 0:
            out["status"][p] = 1
            continue
        st, sc = o.score(ids, req)
        assert st == 0
        fd = sd = 0
        for i, s in zip(ids, sc):
            fd = (fd + mix(2 * int(i) + 1)) & M64
            sd = (sd + mix(2 * int(i) + 2) * (2 * int(s) + 1)) & M64
        out["fit_digest"][p], out["score_digest"][p] = fd, sd
        w = int(ids[int(np.argmax(sc))])
        st, alloc = o.bind(w, req, int(uids[p]))
        out["node"][p], out["status"][p] = w, st
        if st == 0:
            for c, a in enumerate(alloc):
                out["alloc_mask"][p, c] = sum(1 << g for g in a)
    while j < len(mut_at):
        _oracle_mut(o, muts[j]); j += 1
    return out


def _oracle_mut(o, rec):
    kind, node, req, alloc, uid = rec
    if kind == 1:
        o.forget_pod(node, req, alloc, uid)
    else:                                   # ADD, and REPLAY of a uid no podsMap holds: the same row update
        o.add_pod(node, req, alloc, uid)


# ---------------------------------------------------------------------------------------------------- hand cases
def test_ten_gpu_node_from_allocatable_never_uses_gpu_ten_or_above():
    eg = _eg()
    e = eg.Egs(0, 1, 10)
    o = oc.OracleC(0)
    assert e.node_set_allocatable(0, 1000, 10 * 81920) == 0 and o.add_node(1000, 10 * 81920) == 0
    for uid in range(1, 40):
        req = [(int(10 + 7 * uid % 40), 2048, 0)]
        assert list(e.filter([0], req)) == list(o.filter([0], req))
        if e.filter([0], req)[0]:
            st, alloc = e.bind(0, req, uid)
            assert (st, alloc) == o.bind(0, req, uid)
            assert st != 0 or max(alloc[0]) < 10
    assert e.rows(0) == o.rows(0)


@pytest.mark.parametrize("policy", [0, 1])
def test_whole_gpus_and_sentinel_on_a_sixteen_gpu_node(policy):
    eg = _eg()
    e = eg.Egs(policy, 3, 16)
    for i in range(3):
        assert e.node_set(i, 16, 32) == 0
    assert e.bind(0, [(0, 0, 12)], 100)[0] == eg.capi.EGS_ERR_NO_OPTION    # no filter ran: no option (node.go:95)
    assert list(e.filter([0, 1], [(0, 0, 12)])) == [1, 1]
    assert e.bind(0, [(0, 0, 12)], 1) == (0, [list(range(12))])
    assert list(e.filter([1], [(0, 0, 16)])) == [1]
    assert e.bind(1, [(0, 0, 16)], 2) == (0, [list(range(16))])
    assert list(e.filter([0, 1, 2], [(0, 0, 17)])) == [0, 0, 0]
    assert list(e.filter([0], [(0, 0, 5)])) == [0] and list(e.filter([0], [(0, 0, 4)])) == [1]
    e.state_load(2, [0] * 15 + [40], [0] * 15 + [8])
    assert list(e.filter([2], [(-1, -1, 0)])) == [1]
    st, alloc = e.bind(2, [(-1, -1, 0)], 3)
    assert (st, alloc) == (0, [[15]]) and e.rows(2)[15] == (41, 9)


@pytest.mark.parametrize("policy", [0, 1])
def test_score_without_filter_is_the_reference_panic_on_a_wide_node(policy):
    """Score of a node that fits but has no cached option: the reference dereferences a nil option (node.go:84).  The
    option Assume cached on the way stays, with the oracle's masks on GPUs above 8."""
    eg = _eg()
    e = eg.Egs(policy, 2, 16)
    o = oc.OracleC(policy)
    for i, g in enumerate((16, 10)):
        assert e.node_set(i, g, 32) == 0 and o.add_node(100 * g, 32 * g) == i
    e.state_load(0, [0] * 12 + [100] * 4, [0] * 12 + [32] * 4); o.set_rows(0, [0] * 12 + [100] * 4, [0] * 12 + [32] * 4)
    req = [(0, 0, 3)]
    st, sc = e.score([0, 1], req)
    ost, osc = o.score([0, 1], req)
    assert st == ost == eg.capi.EGS_ERR_PANIC and list(sc) == list(osc)
    assert e.peek(0, req) == o.peek(0, req) == ([[12, 13, 14]], o.peek(0, req)[1])
    assert e.peek(1, req) == o.peek(1, req)


# ---------------------------------------------------------------------------------------------------- verb sequences
@pytest.mark.parametrize("policy,seed", [(0, 1), (1, 2), (0, 3)])
def test_seeded_verb_sequences_on_mixed_clusters(policy, seed):
    eg = _eg(); cap = eg.capi
    n = 40
    e, o, rng = _cluster(policy, n, seed)
    gc = [o.gpu_count(i) for i in range(n)]
    uid, bound, seen = 1, [], []
    for step in range(160):
        req = SHAPES[int(rng.integers(len(SHAPES)))]
        if req not in seen:
            seen.append(req)
        k = int(rng.integers(0, 9))
        ids = np.sort(rng.choice(n, size=int(rng.integers(1, n)), replace=False)).astype(np.int32)
        if k <= 1:
            assert list(e.filter(ids, req)) == list(o.filter(ids, req))
        elif k == 2:
            st, sc = e.score(ids, req)
            ost, osc = o.score(ids, req)
            assert st == ost and list(sc) == list(osc)
        elif k <= 4:
            node = int(rng.choice(ids))
            if rng.integers(0, 2):              # make the option stale first: another pod lands on the node
                other = SHAPES[0]
                fit = e.filter([node], other)[0]
                assert fit == o.filter([node], other)[0]
                if fit:
                    assert e.bind(node, other, uid) == o.bind(node, other, uid); uid += 1
            got, want = e.bind(node, req, uid), o.bind(node, req, uid)
            assert got == want, (node, req)
            if got[0] == 0:
                bound.append((node, req, got[1], uid))
            uid += 1
        elif k == 5:
            node = int(rng.choice(ids))
            assert e.peek(node, req) == o.peek(node, req)
        elif k == 6:                            # AddPod of a whole-GPU pod another scheduler placed: 12-index list
            node = int(rng.choice([i for i in range(n) if gc[i] >= 12] or [0]))
            if gc[node] >= 12:
                r = [(0, 0, 12)]; a = [sorted(int(x) for x in rng.choice(gc[node], 12, replace=False))]
                assert e.pod_apply(node, r, a, uid) == o.add_pod(node, r, a, uid) == 0
                bound.append((node, r, a, uid)); uid += 1
        elif k == 7 and bound:                  # ForgetPod
            node, r, a, u = bound.pop(int(rng.integers(len(bound))))
            assert e.pod_cancel(node, r, a, u) == o.forget_pod(node, r, a, u) == 0
            assert e.pod_known(u) == o.known_pod(u) and e.pod_released(u) == o.released_pod(u)
        else:                                   # node replay, then a few mutation records in one launch
            node = int(rng.integers(n))
            r = [(20, 2, 0)]; a = [[int(rng.integers(gc[node]))]]
            L = e.L
            off = np.array([0, 1], np.int32); idx = np.array(a[0], np.int32)
            assert L.egs_node_replay_pod(e.h, node, 1, cap.units_array(r).ctypes.data, off.ctypes.data,
                                         idx.ctypes.data, uid) == 0
            o.add_pod(node, r, a, uid); uid += 1
            recs = []
            for _ in range(3):
                node = int(rng.integers(n))
                if rng.integers(0, 3) == 0 and bound and max(len(x) for x in bound[-1][2]) <= 8:
                    nd, r, a, u = bound.pop()
                    recs.append((cap.EGS_MUT_FORGET, nd, r, a, u))
                else:
                    cnt = int(rng.integers(1, min(gc[node], 8) + 1))
                    r = [(0, 0, cnt)]; a = [sorted(int(x) for x in rng.choice(gc[node], cnt, replace=False))]
                    recs.append((cap.EGS_MUT_ADD, node, r, a, uid)); bound.append((node, r, a, uid)); uid += 1
            assert e.mutations_apply(recs) == 0
            for rec in recs:
                _oracle_mut(o, rec)
        _check_rows(e, o, n)
        _check_caches(e, o, n, seen, rng)
    assert uid > 20


# ---------------------------------------------------------------------------------------------------- batches
def _batch(rng, P):
    c_off, units = [0], []
    for _ in range(P):
        req = SHAPES[int(rng.choice(len(SHAPES), p=_WEIGHTS))]
        units.extend(req); c_off.append(len(units))
    return np.array(c_off, np.int32), np.array(units, np.int32)


_WEIGHTS = np.array([6, 4, 4, 2, 1, 2, 2, 1, 1, 1, 1, 1, 1, 1], float)
_WEIGHTS /= _WEIGHTS.sum()


def test_oracle_driver_matches_the_oracle_batch():
    """The per-pod oracle driver the batch tests use equals egso_schedule_batch on the GPUs the latter can show."""
    n = 60
    _, o1, rng = _cluster(0, n, 21)
    _, o2, _ = _cluster(0, n, 21)
    c_off, units = _batch(rng, 300)
    uids = np.arange(1, 301, dtype=np.uint64)
    a = _oracle_batch(o1, n, c_off, units, uids)
    b = o2.schedule_batch(c_off, units.astype(np.int64), uids=uids)
    for f in FIELDS:
        want = b[f]
        got = (a[f] & 0xFF).astype(np.uint8) if f == "alloc_mask" else a[f]
        assert np.array_equal(got, want), f


@pytest.mark.parametrize("policy", [0, 1])
def test_batches_on_a_mixed_cluster(policy):
    import torch
    eg = _eg(); cap = eg.capi
    n, P = 120, 400
    _, o, rng = _cluster(policy, n, 100 + policy)
    c_off, units = _batch(rng, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    ref = _oracle_batch(o, n, c_off, units, uids)
    shapes = eg.workloads.shapes_of(eg.workloads.Workload(0, n, 16, 0, policy, None, None, c_off, units))
    shapes = [list(s) for s in shapes]

    def check(e, got):
        for f in FIELDS:
            assert np.array_equal(got[f], ref[f]), f"{f} differs at pod {np.argwhere(got[f] != ref[f])[:3]}"
        _check_rows(e, o, n)
        _check_caches(e, o, n, shapes, rng)

    e, _, _ = _cluster(policy, n, 100 + policy)
    check(e, e.schedule_batch(c_off, units, uids=uids))                       # AUTO: the per-pod engine
    assert all(e.pod_known(int(u)) == o.known_pod(int(u)) for u in uids[:50])

    e, _, _ = _cluster(policy, n, 100 + policy)
    got = e.schedule_batch_vec(c_off, units, 40, uids=uids)
    check(e, got)
    _, o2, _ = _cluster(policy, n, 100 + policy)
    for p in range(40):                                                        # the full vectors, element-wise
        req = _req(units, c_off, p)
        fit = o2.filter(None, req)
        assert np.array_equal(got["vec_fit"][p], fit), p
        ids = np.flatnonzero(fit).astype(np.int32)
        sc = np.zeros(n, np.int32)
        if len(ids):
            sc[ids] = o2.score(ids, req)[1]
        assert np.array_equal(got["vec_score"][p], sc), p
        if ref["node"][p] >= 0:
            o2.bind(int(ref["node"][p]), req, int(uids[p]))

    e, _, _ = _cluster(policy, n, 100 + policy)
    dev = [torch.zeros(P, dtype=torch.int32, device="cuda"), torch.zeros(P, dtype=torch.int32, device="cuda"),
           torch.zeros(P * 8, dtype=torch.uint8, device="cuda"), torch.zeros(P, dtype=torch.int32, device="cuda"),
           torch.zeros(P, dtype=torch.int64, device="cuda"), torch.zeros(P, dtype=torch.int64, device="cuda")]
    e.schedule_batch_device(c_off, units, [t.data_ptr() for t in dev])
    torch.cuda.synchronize()
    got = dict(node=dev[0].cpu().numpy(), status=dev[1].cpu().numpy(),
               alloc_mask=dev[2].cpu().numpy().view("<u2").reshape(P, 4), fit_count=dev[3].cpu().numpy(),
               fit_digest=dev[4].cpu().numpy().view(np.uint64), score_digest=dev[5].cpu().numpy().view(np.uint64))
    lib_uid = 0x8000000000000000                                                # the library numbers these pods
    _, o3, _ = _cluster(policy, n, 100 + policy)
    ref3 = _oracle_batch(o3, n, c_off, units, np.arange(lib_uid, lib_uid + P, dtype=np.uint64))
    for f in FIELDS:
        assert np.array_equal(got[f], ref3[f]), f
    _check_rows(e, o3, n)


@pytest.mark.parametrize("policy", [0, 1])
def test_batch_with_mutations_woven_in(policy):
    eg = _eg(); cap = eg.capi
    n, P = 100, 300
    e, o, rng = _cluster(policy, n, 200 + policy)
    gc = [o.gpu_count(i) for i in range(n)]
    c_off, units = _batch(rng, P)
    uids = np.arange(1, P + 1, dtype=np.uint64)
    mut_at = sorted(int(x) for x in rng.integers(0, P + 1, 40))
    recs = []
    for j in range(len(mut_at)):
        node = int(rng.integers(n))
        if j % 4 == 3:
            kind, node, r, a, u = recs[-1]
            recs.append((cap.EGS_MUT_FORGET, node, r, a, u))
        else:
            cnt = int(rng.integers(1, min(gc[node], 8) + 1))
            r = [(0, 0, cnt)] if j % 2 else [(int(rng.choice([10, 30])), 2, 0)]
            a = [sorted(int(x) for x in rng.choice(gc[node], cnt if j % 2 else 1, replace=False))]
            recs.append((cap.EGS_MUT_ADD, node, r, a, 1_000_000 + j))
    got = e.schedule_batch_mut(c_off, units, mut_at, recs, uids=uids)
    ref = _oracle_batch(o, n, c_off, units, uids, recs, mut_at)
    for f in FIELDS:
        assert np.array_equal(got[f], ref[f]), f"{f} differs at pod {np.argwhere(got[f] != ref[f])[:3]}"
    _check_rows(e, o, n)
    _check_caches(e, o, n, [list(s) for s in SHAPES], rng)


# ---------------------------------------------------------------------------------------------------- guards
def test_guards_of_a_wide_handle():
    eg = _eg(); cap = eg.capi
    with pytest.raises(cap.EgsError):
        eg.Egs(0, 4, 17)
    e, o, rng = _cluster(0, 8, 5, gs=[9, 16])
    assert e.node_set_allocatable(0, 1700, 17 * 16) == cap.EGS_ERR_BAD_ARG
    assert e.node_set(0, 17, 16) == cap.EGS_ERR_BAD_ARG
    assert e.node_set(0, 12, (1 << 25) + 1) == cap.EGS_ERR_OVERFLOW_GUARD
    assert e.state_load(1, [1 << 20] * o.gpu_count(1), [(1 << 25) + 1] * o.gpu_count(1)) == cap.EGS_ERR_OVERFLOW_GUARD
    with pytest.raises(cap.EgsError):
        e.filter([0], [(10, (1 << 25) + 1, 0)])
    before = e.state_dump()
    c_off, units = np.array([0, 1, 2], np.int32), np.array([[10, 1, 0], [0, 0, 2]], np.int32)
    with pytest.raises(cap.EgsError) as ex:
        e.schedule_batch(c_off, units, uids=np.array([7, 8], np.uint64), mode=cap.EGS_MODE_ROUNDS)
    assert ex.value.status == cap.EGS_ERR_BAD_ARG and "ROUNDS" in str(ex.value)
    rec = [(cap.EGS_MUT_ADD, 0, [(0, 0, 1)], [[0]], 99)]
    with pytest.raises(cap.EgsError) as ex:
        e.schedule_batch_mut(c_off, units, [0], rec, mode=cap.EGS_MODE_ROUNDS)
    assert ex.value.status == cap.EGS_ERR_BAD_ARG
    with pytest.raises(cap.EgsError) as ex:
        e.shard_set(0, 2)
    assert ex.value.status == cap.EGS_ERR_BAD_ARG and "rounds" in str(ex.value)
    a = cap.mutations_array([(cap.EGS_MUT_ADD, 0, [(0, 0, 9)], [list(range(8))], 98)])
    a[0]["n_idx"][0] = 9                                             # nine indices: more than a record holds
    assert e.L.egs_mutations_apply(e.h, 1, cap._p(a)) == cap.EGS_ERR_BAD_ARG
    after = e.state_dump()
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    assert not e.pod_known(7) and not e.pod_known(99) and not e.pod_known(98)
    # the int32 guard on a 16-GPU node: values at 2^20 / 2^25 Trade exactly as the oracle (int64)
    assert e.node_set(2, 16, 1 << 25) == 0 and o.add_node(1600, 16 << 25) == 8
    core = [1 << 20] * 15 + [100]; mem = [1 << 25] * 15 + [1 << 25]
    e.state_load(2, core, mem); o.set_rows(8, core, mem)
    for req in ([(99, 1 << 25, 0)], [(0, 0, 1)], [(1 << 20, 0, 0)]):
        assert list(e.filter([2], req)) == list(o.filter([8], req))
        assert e.peek(2, req) == o.peek(8, req)


# ---------------------------------------------------------------------------------------------------- engines
def test_per_pod_engine_on_a_wide_handle_equals_the_rounds_engine():
    """The same 8-GPU config-4-style cluster and batch: rounds engine on a g_max = 8 handle, per-pod engine on a wide
    handle.  Same outputs (masks widened to u16) and the same rows."""
    eg = _eg(); cap = eg.capi
    w = eg.workloads.config(4, n_nodes=20_000, n_pods=200_000)
    got = []
    for g_max in (8, 16):
        e = eg.Egs(w.policy, w.n_nodes, g_max)
        e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
        got.append((e.schedule_batch(w.c_off, w.units), e.state_dump()[:2]))
        e.close()
    (a, rows_a), (b, rows_b) = got
    assert a["alloc_mask"].dtype == np.uint8 and b["alloc_mask"].dtype == np.uint16
    for f in FIELDS:
        assert np.array_equal(a[f].astype(np.uint16) if f == "alloc_mask" else a[f], b[f]), f
    assert np.array_equal(rows_a[0], rows_b[0][:, :8]) and np.array_equal(rows_a[1], rows_b[1][:, :8])
    assert (rows_b[0][:, 8:] == cap.EGS_PAD).all()
    assert (a["status"] == 0).any()


def test_device_batch_refuses_a_misaligned_mask_buffer():
    """A wide handle stores each pod's four u16 masks as one 8-byte word: a buffer that is not 8-byte aligned is
    refused before anything runs."""
    import torch
    eg = _eg(); cap = eg.capi
    e = eg.Egs(0, 4, 16)
    for i in range(4):
        assert e.node_set(i, 16, 32) == 0
    c_off, units = np.array([0, 1], np.int32), np.array([[10, 4, 0]], np.int32)
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    with pytest.raises(cap.EgsError) as ex:
        e.schedule_batch_device(c_off, units, [0, 0, buf.data_ptr() + 4, 0, 0, 0])
    assert ex.value.status == cap.EGS_ERR_BAD_ARG
    assert e.rows(0) == [(100, 32)] * 16
    e.schedule_batch_device(c_off, units, [0, 0, buf.data_ptr() + 8, 0, 0, 0])
    torch.cuda.synchronize()
    assert buf.cpu().numpy()[8:16].view("<u2")[0] == 1 << 15 and e.rows(0)[15] == (90, 28)   # first node of the tie
