"""egs_checkpoint_save / _rollback / _drop against the C oracle: a rollback after any sequence of verbs returns every
answer to what it was at the save; a dry run equals the real run that follows it on every engine and on an in-process
shard group; the stale cached option a ForgetPod loses comes back; all-or-nothing admission of pod groups; and the
guards."""
import threading

import numpy as np
import pytest

import oracle_c as oc
from oracle_harness import Cluster, compare_caches, compare_outputs, compare_rows, egs, oracle_batch

pytestmark = pytest.mark.gpu

LIB = 0x8000000000000000                    # the first library-assigned uid
SHAPES = [
    [(10, 4, 0)], [(50, 8, 0)], [(25, 2, 0)], [(0, 6, 0)], [(-1, -1, 0)],
    [(0, 0, 1)], [(0, 0, 2)], [(0, 0, 4)], [(30, 2, 0), (0, 0, 2)], [(20, 4, 0), (-1, -1, 0), (10, 1, 0)],
]
LATE = [[(15, 3, 0)], [(0, 0, 3)], [(40, 3, 0), (40, 3, 0)]]     # interned only inside a what-if
WIDE_SHAPES = [[(0, 0, 12)], [(0, 0, 9), (5, 1, 0)]]


def _cluster(policy, n, seed, g_max):
    """n nodes of 1..g_max GPUs, about half of them partly used; and the rng that drew them."""
    rng = np.random.default_rng(seed)
    gs = [1, 2, 4, 8] if g_max == 8 else [1, 2, 8, 9, 12, 16]
    nodes = []
    for _ in range(n):
        G = int(rng.choice(gs)); M = int(rng.choice([16, 32]))
        rows = None
        if rng.integers(0, 2):
            core = [100 if rng.integers(0, 3) == 0 else int(rng.integers(0, 101)) for _ in range(G)]
            rows = (core, [M if c == 100 else int(rng.integers(0, M + 1)) for c in core])
        nodes.append((G, M, rows))
    return Cluster(policy, nodes, g_max), rng


def _batch(rng, P, shapes):
    c_off, units = [0], []
    for _ in range(P):
        units.extend(shapes[int(rng.integers(len(shapes)))]); c_off.append(len(units))
    return np.array(c_off, np.int32), np.array(units, np.int32)


def _state(e, shapes, uids):
    """Every answer the round trip compares: rows with gpu_count / mem_total, option dumps, uid maps."""
    return (e.state_dump(), [e.option_dump(s) for s in shapes],
            {int(u): (e.pod_known(int(u)), e.pod_released(int(u))) for u in uids})


def _assert_same_state(a, b, what):
    """b equals a; a uid that a does not hold was never used before a was taken: unknown, not released."""
    for x, y in zip(a[0], b[0]):
        assert x.tobytes() == y.tobytes(), f"{what}: state_dump"
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        for u, v in zip(x, y):
            assert u.tobytes() == v.tobytes(), f"{what}: option_dump of shape {i}"
    for u, got in b[2].items():
        assert got == a[2].get(u, (False, False)), f"{what}: pod_known / pod_released of {hex(u)}"


# ------------------------------------------------------------------------------------------- 1. every verb
def _what_if(e, rng, n, uid, touched):
    """A random sequence of every state-changing verb, answers unchecked.  Returns the next free uid."""
    import torch
    cap = egs().capi
    shapes = SHAPES + LATE + (WIDE_SHAPES if e.g_max > 8 else [])
    modes = [cap.EGS_MODE_AUTO, cap.EGS_MODE_RESCAN] + ([cap.EGS_MODE_ROUNDS] if e.g_max <= 8 else [])
    gc = lambda node: int(e.state_dump(node, 1)[2][0])
    for _ in range(int(rng.integers(12, 24))):
        req = shapes[int(rng.integers(len(shapes)))]
        node = int(rng.integers(n))
        k = int(rng.integers(0, 14))
        if k == 0:
            e.filter(None, req)
        elif k == 1:
            e.score(np.flatnonzero(e.filter(None, req)).astype(np.int32), req)
        elif k == 2:
            e.filter([node], req); e.bind(node, req, uid); touched.add(uid); uid += 1
        elif k == 3:
            g = gc(node); a = [[int(rng.integers(g))]]
            e.pod_apply(node, [(20, 2, 0)], a, uid); touched.add(uid); uid += 1
        elif k == 4:
            g = gc(node); a = [[int(rng.integers(g))]]
            off, idx = np.array([0, 1], np.int32), np.array(a[0], np.int32)
            e.L.egs_node_replay_pod(e.h, node, 1, cap.units_array([(10, 1, 0)]).ctypes.data, off.ctypes.data,
                                    idx.ctypes.data, uid)
            touched.add(uid); uid += 1
        elif k == 5 and touched:
            u = int(rng.choice(sorted(touched)))
            e.pod_cancel(int(rng.integers(-1, n)), [(20, 2, 0)], [[0]], u)
        elif k == 6:
            g = gc(node)
            recs = [(cap.EGS_MUT_ADD, node, [(0, 0, 1)], [[int(rng.integers(g))]], uid),
                    (cap.EGS_MUT_FORGET, node, [(0, 0, 1)], [[0]], int(rng.choice(sorted(touched | {uid}))))]
            e.mutations_apply(recs); touched.add(uid); uid += 1
        elif k == 7:
            c_off, units = _batch(rng, int(rng.integers(1, 40)), shapes)
            P = len(c_off) - 1
            uids = None
            if rng.integers(0, 2):
                uids = np.arange(uid, uid + P, dtype=np.uint64); touched.update(int(u) for u in uids); uid += P
            e.schedule_batch(c_off, units, uids=uids, mode=int(rng.choice(modes)))
        elif k == 8:
            c_off, units = _batch(rng, 20, shapes)
            g = gc(node)
            recs = [(cap.EGS_MUT_ADD, node, [(0, 0, 1)], [[int(rng.integers(g))]], uid)]
            touched.add(uid); uid += 1
            e.schedule_batch_mut(c_off, units, [int(rng.integers(0, 21))], recs, mode=int(rng.choice(modes)))
        elif k == 9:
            c_off, units = _batch(rng, 10, shapes)
            e.schedule_batch_vec(c_off, units, 3)
        elif k == 10:
            c_off, units = _batch(rng, 16, shapes)
            dev = [torch.zeros(16, dtype=torch.int32, device="cuda"), torch.zeros(16, dtype=torch.int32, device="cuda"),
                   torch.zeros(16 * 8, dtype=torch.uint8, device="cuda")]
            e.schedule_batch_device(c_off, units, [d.data_ptr() for d in dev] + [0, 0, 0])
            torch.cuda.synchronize()
        elif k == 11:
            G = int(rng.integers(1, e.g_max + 1))
            e.node_set_allocatable(node, 100 * G, 16 * G)
        elif k == 12:
            g = gc(node)
            if rng.integers(0, 2):
                e.state_load(node, [int(x) for x in rng.integers(0, 101, g)], [int(x) for x in rng.integers(0, 17, g)])
            else:
                m = int(rng.integers(1, 4)); n0 = min(node, n - m); G = int(rng.integers(1, e.g_max + 1))
                e.state_load_bulk(n0, G, 32, np.full((m, G), 100, np.int32), np.full((m, G), 32, np.int32))
        else:
            e.restore()
    return uid


@pytest.mark.parametrize("g_max,policy,seed", [(8, 0, 1), (8, 1, 2), (16, 0, 3), (16, 1, 4)])
def test_round_trip_over_every_verb(g_max, policy, seed):
    n, P = 40, 120
    cl, rng = _cluster(policy, n, seed, g_max)
    early = SHAPES + (WIDE_SHAPES if g_max > 8 else [])
    hist = _batch(rng, P, early)
    last = _batch(rng, 60, early)
    e, twin = cl.handle(), cl.handle()
    for h in (e, twin):
        h.snapshot()                                        # the what-if may restore to it: a copy, not state
        h.schedule_batch(*hist)                             # library uids LIB .. LIB+P-1
        h.filter(None, early[0])
    touched = set(range(LIB, LIB + P + 1000)) | {1, 2, 3}   # and the library uids a what-if assigns
    before = _state(e, early, touched)
    e.checkpoint_save()
    uid = 1000
    for trial in range(3):                                  # three what-ifs from the one checkpoint
        touched = set(touched)
        uid = _what_if(e, rng, n, uid, touched)
        e.checkpoint_rollback()
        _assert_same_state(before, _state(e, early, touched), f"what-if {trial}")
        for s in LATE:                                      # interned after the save: forgotten, all ABSENT again
            st, sc, am = e.option_dump(s)
            assert not st.any() and not sc.any() and not am.any(), f"what-if {trial}: shape {s} after the rollback"
    # one more batch: the same outputs as the twin that never ran a what-if, and as the oracle
    got, ref_twin = e.schedule_batch(*last), twin.schedule_batch(*last)
    compare_outputs(ref_twin, got, "after the what-ifs vs the twin")
    o = cl.oracle()
    oracle_batch(o, *hist, np.arange(LIB, LIB + P, dtype=np.uint64))
    o.filter(None, early[0])
    ref = oracle_batch(o, *last, np.arange(LIB + P, LIB + P + 60, dtype=np.uint64))
    compare_outputs(ref, got, "after the what-ifs vs the oracle")
    compare_rows(e, o, range(n))
    compare_caches(e, o, early, range(n), unfit_check=True)
    for u in sorted(touched | set(range(LIB + P, LIB + P + 60))):
        assert (e.pod_known(u), e.pod_released(u)) == (o.known_pod(u), o.released_pod(u)), hex(u)


# ------------------------------------------------------------------------------------------- 2. dry run
def _modes(g_max):
    cap = egs().capi
    return [cap.EGS_MODE_AUTO, cap.EGS_MODE_RESCAN] + ([cap.EGS_MODE_ROUNDS] if g_max <= 8 else [])


@pytest.mark.parametrize("g_max", [8, 16])
@pytest.mark.parametrize("explicit", [False, True])
def test_dry_run_equals_the_real_run(g_max, explicit):
    n, P = 80, 300
    for mode in _modes(g_max):
        cl, rng = _cluster(1, n, 40 + g_max, g_max)
        c_off, units = _batch(rng, P, SHAPES + (WIDE_SHAPES if g_max > 8 else []))
        uids = np.arange(5000, 5000 + P, dtype=np.uint64) if explicit else None
        want_uids = uids if explicit else np.arange(LIB, LIB + P, dtype=np.uint64)
        e, o = cl.handle(), cl.oracle()
        ref = oracle_batch(o, c_off, units, want_uids)
        e.checkpoint_save()
        dry = e.schedule_batch(c_off, units, uids=uids, mode=mode)
        ok = want_uids[dry["status"] == 0]
        assert ok.size and all(e.pod_known(int(u)) for u in ok[:20])
        e.checkpoint_rollback()
        assert not any(e.pod_known(int(u)) for u in ok[:20]), f"mode {mode}: the dry run's uids stay known"
        real = e.schedule_batch(c_off, units, uids=uids, mode=mode)    # explicit: the dry run's uids are free again
        compare_outputs(dry, real, f"mode {mode}: dry vs real")
        compare_outputs(ref, real, f"mode {mode}: real vs oracle")
        compare_rows(e, o, range(n))
        assert all(e.pod_known(int(u)) for u in ok[:20])
        if explicit:                                        # without the rollback the same uids are refused
            with pytest.raises(egs().capi.EgsError):
                e.schedule_batch(c_off, units, uids=uids, mode=mode)
        e.close()


@pytest.mark.parametrize("world", [2, 4])
def test_dry_run_on_a_shard_group(world):
    cap = egs().capi
    w = egs().workloads.config(4, n_nodes=4096, n_pods=20_000)
    cl = Cluster.of_workload(w)
    P = len(w.c_off) - 1
    o = cl.oracle()
    ref = o.schedule_batch(w.c_off, w.units.astype(np.int64), uids=np.arange(LIB, LIB + P, dtype=np.uint64))
    hs = [cl.handle(world, r) for r in range(world)]
    cap.comm_init_local(hs)
    outs, errs = [None] * world, []

    def run(r):
        try:
            h = hs[r]
            h.checkpoint_save()
            dry = h.schedule_batch(w.c_off, w.units, mode=cap.EGS_MODE_ROUNDS)
            h.checkpoint_rollback()
            outs[r] = (dry, h.schedule_batch(w.c_off, w.units, mode=cap.EGS_MODE_ROUNDS))
        except Exception as ex:   # pragma: no cover
            errs.append(repr(ex))
    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join(timeout=600)
    assert not errs, errs
    for r, h in enumerate(hs):
        dry, real = outs[r]
        compare_outputs(dry, real, f"rank {r}: dry vs real")
        compare_outputs(ref, real, f"rank {r}: real vs oracle")
        lo, hi = cap.shard_range(h.max_nodes, r, world)
        core, mem = h.state_dump(lo, hi - lo)[:2]
        for i in range(lo, hi):
            assert list(zip(core[i - lo, :8].tolist(), mem[i - lo, :8].tolist())) == o.rows(i), f"rank {r}: node {i}"
        assert h.pod_known(LIB) == o.known_pod(LIB)
        h.close()


# ------------------------------------------------------------------------------------------- 3. the stale option
def test_rollback_keeps_the_stale_option_a_forget_loses():
    """Spread policy, one node of two empty GPUs.  Filter caches pod A's option on GPU 1 (the last maximal leaf,
    gpu.go:85); pod B then lands on GPU 1 and leaves too little there for A, so the cached option is stale.  A bind
    of A consumes it, deletes it (node.go:90-92) and fails in Transact.  ForgetPod of that pod gives back nothing and
    not the option either: the next pod of A's shape Trades fresh and binds on GPU 0.  A rollback instead of the
    ForgetPod brings the stale option back: the next pod takes it and fails again, as in the oracle where the first
    bind never happened."""
    cap = egs().capi
    A, B = [(50, 8, 0)], [(60, 4, 0)]

    def setup(h, oracle):
        if oracle:
            h.add_node(200, 32)
        else:
            assert h.node_set(0, 2, 16) == 0
        assert list(h.filter([0], A)) == [1] and list(h.filter([0], B)) == [1]
        assert h.bind(0, B, 1) == (0, [[1]])
        assert list(h.filter([0], A)) == [1]                # a cache hit: the stale option

    eg = egs()
    forget, back = eg.Egs(1, 1, 8), eg.Egs(1, 1, 8)
    setup(forget, False); setup(back, False)
    first = forget.bind(0, A, 2)
    assert first == (cap.EGS_ERR_TRANSACT, None)
    assert forget.pod_cancel(0, A, [[]], 2) == 0
    forget.filter([0], A)
    after_forget = (forget.bind(0, A, 3), forget.rows(0))
    back.checkpoint_save()
    assert back.bind(0, A, 2) == first
    back.checkpoint_rollback()
    back.filter([0], A)
    after_rollback = (back.bind(0, A, 3), back.rows(0))

    o = oc.OracleC(1)                                       # the history without the first bind
    setup(o, True)
    o.filter([0], A)
    assert after_rollback == (o.bind(0, A, 3), o.rows(0)) == ((cap.EGS_ERR_TRANSACT, None), [(100, 16), (40, 12)])
    o = oc.OracleC(1)                                       # the history with the bind and the ForgetPod
    setup(o, True)
    o.bind(0, A, 2); o.forget_pod(0, A, [[]], 2); o.filter([0], A)
    assert after_forget == (o.bind(0, A, 3), o.rows(0)) == ((0, [[0]]), [(50, 8), (40, 12)])
    assert after_forget != after_rollback


# ------------------------------------------------------------------------------------------- 4. gangs
GANG_SHAPES = [[(0, 0, 1)], [(0, 0, 2)], [(0, 0, 4)], [(-1, -1, 0)], [(40, 8, 0)],
               [(30, 2, 0), (0, 0, 1)], [(20, 4, 0), (-1, -1, 0), (10, 1, 0)]]


@pytest.mark.parametrize("g_max,seed", [(8, 7), (16, 8)])
def test_gang_admission_all_or_nothing(g_max, seed):
    n = 12
    cl, rng = _cluster(0, n, seed, g_max)
    e = cl.handle()
    groups, admitted, uid = [], [], 1
    for _ in range(40):
        k = int(rng.integers(1, 9))
        reqs = [GANG_SHAPES[int(rng.integers(len(GANG_SHAPES)))] for _ in range(k)]
        units = [u for r in reqs for u in r]
        c_off = np.cumsum([0] + [len(r) for r in reqs]).astype(np.int32)
        groups.append((c_off, np.array(units, np.int32), np.arange(uid, uid + k, dtype=np.uint64)))
        uid += k
    for gi, (c_off, units, uids) in enumerate(groups):
        e.checkpoint_save()
        out = e.schedule_batch(c_off, units, uids=uids)
        ok = bool((out["status"] == 0).all())
        if not ok:
            e.checkpoint_rollback()
        o = cl.oracle()                                     # the oracle's decision: admitted prefix + this group
        for j in admitted:
            oracle_batch(o, *groups[j])
        want = bool((oracle_batch(o, c_off, units, uids)["status"] == 0).all())
        assert ok == want, f"group {gi}"
        if ok:
            admitted.append(gi)
    e.checkpoint_drop()
    assert 0 < len(admitted) < len(groups)
    o = cl.oracle()
    for j in admitted:
        oracle_batch(o, *groups[j])
    compare_rows(e, o, range(n))
    compare_caches(e, o, GANG_SHAPES, range(n), unfit_check=True)
    for c_off, units, uids in groups:
        for u in uids:
            assert (e.pod_known(int(u)), e.pod_released(int(u))) == (o.known_pod(int(u)), o.released_pod(int(u)))


# ------------------------------------------------------------------------------------------- 5. guards
def test_repeated_rollback_replace_and_guards():
    cap = egs().capi
    cl, rng = _cluster(0, 30, 9, 8)
    e = cl.handle()
    with pytest.raises(cap.EgsError) as ex:                 # no checkpoint yet
        e.checkpoint_rollback()
    assert ex.value.status == cap.EGS_ERR_BAD_ARG and "checkpoint" in str(ex.value)
    b1, b2 = _batch(rng, 50, SHAPES), _batch(rng, 50, SHAPES)
    e.schedule_batch(*b1)
    e.checkpoint_save()
    s1 = _state(e, SHAPES, range(LIB, LIB + 100))
    outs = []
    for _ in range(3):                                      # several rollbacks from one checkpoint
        outs.append(e.schedule_batch(*b2))
        e.checkpoint_rollback()
        _assert_same_state(s1, _state(e, SHAPES, range(LIB, LIB + 100)), "repeated rollback")
    compare_outputs(outs[0], outs[1], "second what-if"); compare_outputs(outs[0], outs[2], "third what-if")
    e.schedule_batch(*b2)
    e.checkpoint_save()                                     # replaces the first checkpoint
    s2 = _state(e, SHAPES, range(LIB, LIB + 100))
    e.schedule_batch(*b1)
    e.checkpoint_rollback()
    _assert_same_state(s2, _state(e, SHAPES, range(LIB, LIB + 100)), "second save")
    e.checkpoint_drop()
    with pytest.raises(cap.EgsError) as ex:                 # dropped: nothing to return to, nothing changes
        e.checkpoint_rollback()
    assert ex.value.status == cap.EGS_ERR_BAD_ARG
    _assert_same_state(s2, _state(e, SHAPES, range(LIB, LIB + 100)), "rollback after drop")
    e.checkpoint_drop()                                     # dropping nothing is fine
    e.checkpoint_save()
    e.shard_set(0, 1)                                       # a new shard layout drops the checkpoint
    with pytest.raises(cap.EgsError) as ex:
        e.checkpoint_rollback()
    assert ex.value.status == cap.EGS_ERR_BAD_ARG
    e.checkpoint_save()
    e.close()                                               # destroy frees an open checkpoint
