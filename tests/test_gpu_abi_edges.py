"""Edge cases of the C ABI on the GPU: argument guards, int32 overflow guards, node replay,
snapshot/restore, status of unknown nodes, uid rules of the batch call."""
import numpy as np
import pytest

import oracle_c as oc
from oracle_harness import Cluster, compare_outputs, egs

pytestmark = pytest.mark.gpu


def test_guards_and_bad_arguments():
    eg = egs(); cap = eg.capi
    e = eg.Egs(0, 8)
    assert e.node_set_allocatable(0, 99, 10) == cap.EGS_ERR_NO_GPU            # node.go:28-30
    assert e.node_set_allocatable(0, 900, 10) == cap.EGS_ERR_BAD_ARG          # more GPUs than the row holds
    assert e.node_set(0, 4, (1 << 25) + 1) == cap.EGS_ERR_OVERFLOW_GUARD      # int32-exact range
    assert e.node_set(9, 4, 16) == cap.EGS_ERR_BAD_ARG
    assert e.node_set(0, 4, 16) == 0
    assert e.state_load(1, [100] * 4, [16] * 4) == cap.EGS_ERR_NO_NODE        # never set
    assert e.state_load(0, [100, 100, 100, -1], [16] * 4) == cap.EGS_ERR_OVERFLOW_GUARD
    with pytest.raises(cap.EgsError):
        e.filter([0], [(10, 1, 0)] * 5)                                       # more than EGS_MAX_CONTAINERS
    with pytest.raises(cap.EgsError):
        e.filter([0], [(-2, 1, 0)])
    assert list(e.filter([0, 1, 7, -3, 99], [(10, 1, 0)])) == [1, 0, 0, 0, 0]  # unknown / out of range ids: unfit
    st, sc = e.score([1, 99], [(10, 1, 0)])
    assert st == 0 and list(sc) == [0, 0]                                     # ScoreMin, scheduler.go:176-179
    assert e.bind(1, [(10, 1, 0)], 1)[0] == cap.EGS_ERR_NO_NODE
    assert e.pod_apply(0, [(0, 0, 1)], [[7]], 5) == cap.EGS_ERR_BAD_ARG       # GPU index out of range (Go would panic)
    vec_fit, vec_score = np.zeros(8, np.uint8), np.zeros(8, np.int32)
    assert e.L.egs_schedule_batch_vec(e.h, -1, None, None, None, 1, cap._p(vec_fit), cap._p(vec_score),
                                      *[None] * 6) == cap.EGS_ERR_BAD_ARG     # n_pods < 0, before any vector is sized


def test_whole_gpu_larger_than_node_and_sentinel_only():
    eg = egs()
    e = eg.Egs(0, 2)
    assert e.node_set_allocatable(0, 200, 32) == 0
    assert list(e.filter([0], [(0, 0, 3)])) == [0]                            # 3 whole GPUs on a 2-GPU node
    assert list(e.filter([0], [(0, 0, 2)])) == [1]
    st, alloc = e.bind(0, [(0, 0, 2)], 1)
    assert st == 0 and alloc == [[0, 1]] and e.rows(0) == [(0, 0), (0, 0)]
    assert list(e.filter([0], [(-1, -1, 0)])) == [1]                          # sentinel fits anything >= -1 (gpu.go:55)
    st, alloc = e.bind(0, [(-1, -1, 0)], 2)
    assert st == 0 and alloc == [[1]] and e.rows(0) == [(0, 0), (1, 1)]       # and ADDS 1 (gpu.go:36-37)


def test_node_replay_then_addpod_is_idempotent():
    eg = egs()
    e = eg.Egs(0, 2)
    e.node_set_allocatable(0, 400, 64)
    off = np.array([0, 1], np.int32); idx = np.array([2, 0], np.int32)
    u = eg.capi.units_array([(30, 4, 0)])
    L = e.L
    assert L.egs_node_replay_pod(e.h, 0, 1, u.ctypes.data, off.ctypes.data, idx.ctypes.data, 77) == 0
    assert e.rows(0)[2] == (70, 12) and not e.pod_known(77)                    # node-level only (node.go:148-160)
    assert L.egs_node_replay_pod(e.h, 0, 1, u.ctypes.data, off.ctypes.data, idx.ctypes.data, 77) == 0
    assert e.rows(0)[2] == (70, 12)                                            # same uid: no-op
    assert e.pod_apply(0, [(30, 4, 0)], [[2]], 77) == 0                        # informer AddPod: podsMap already has it
    assert e.rows(0)[2] == (70, 12) and e.pod_known(77)
    assert e.pod_cancel(0, [(30, 4, 0)], [[2]], 77) == 0
    assert e.rows(0)[2] == (100, 16) and e.pod_released(77) and not e.pod_known(77)


def test_snapshot_restore_and_uid_rules():
    eg = egs(); cap = eg.capi
    w = eg.workloads.config(1, n_nodes=64, n_pods=300)
    e = Cluster.of_workload(w).handle()
    e.snapshot()
    a = e.schedule_batch(w.c_off, w.units, mode=cap.EGS_MODE_ROUNDS)
    rows_a = e.state_dump()[:2]
    assert e.pod_known(0x8000000000000000)                                     # library-assigned uids
    e.restore()
    assert not e.pod_known(0x8000000000000000)
    core, mem, _, _ = e.state_dump()
    assert np.array_equal(core[:, :8], w.core) and np.array_equal(mem[:, :8], w.mem)
    compare_outputs(a, e.schedule_batch(w.c_off, w.units, mode=cap.EGS_MODE_RESCAN), "rescan after restore")
    assert all(np.array_equal(x, y) for x, y in zip(rows_a, e.state_dump()[:2]))
    uids = np.arange(1000, 1300, dtype=np.uint64)
    e.restore()
    e.schedule_batch(w.c_off, w.units, uids=uids)
    assert e.pod_known(1000)
    with pytest.raises(cap.EgsError):
        e.schedule_batch(w.c_off, w.units, uids=uids)                          # already known uids
    dup = uids.copy(); dup[5] = dup[4]; dup += 5000
    with pytest.raises(cap.EgsError):
        e.schedule_batch(w.c_off, w.units, uids=dup)


def test_mode_switching_keeps_state_consistent():
    """rounds -> verbs -> rescan -> rounds on one handle equals the oracle doing the same sequence."""
    eg = egs(); cap = eg.capi
    w = eg.workloads.config(4, n_nodes=48, n_pods=900)
    cl = Cluster.of_workload(w)
    e, o = cl.handle(), cl.oracle()
    u64 = w.units64()
    for lo, hi, mode in [(0, 300, cap.EGS_MODE_ROUNDS), (300, 600, cap.EGS_MODE_RESCAN), (600, 900, cap.EGS_MODE_ROUNDS)]:
        off = w.c_off[lo:hi + 1] - w.c_off[lo]
        ref = o.schedule_batch(off, u64[w.c_off[lo]:w.c_off[hi]], uids=np.arange(lo, hi, dtype=np.uint64))
        got = e.schedule_batch(off, w.units[w.c_off[lo]:w.c_off[hi]], uids=np.arange(lo, hi, dtype=np.uint64), mode=mode)
        compare_outputs(ref, got, f"pods from {lo}")
        req = [tuple(int(x) for x in w.units[w.c_off[hi - 1]])]
        assert list(e.filter(None, req)) == list(o.filter(None, req))          # verbs see the tables the batch left
        assert list(e.score(None, req)[1]) == [int(x) for x in o.score(None, req)[1]]


def test_node_reload_after_auto_uid_batch_drops_pods_map():
    """A batch with library-assigned uids keeps podsMap membership in the batch's result arrays; reloading the node
    (a fresh NodeAllocator, node.go:42-50) must drop it all the same: a later ForgetPod of such a uid is a no-op on
    the rows (node.go:131) and a bind with that uid transacts again (node.go:149)."""
    eg = egs()
    e = eg.Egs(0, 1)
    e.node_set_allocatable(0, 200, 32)
    c_off = np.array([0, 1], np.int32)
    units = np.array([[20, 4, 0]], np.int32)
    out = e.schedule_batch(c_off, units, mode=2)                                # uids == NULL: library-assigned
    assert out["status"][0] == 0 and out["node"][0] == 0
    uid = 0x8000000000000000
    assert e.pod_known(uid)
    g = int(np.log2(out["alloc_mask"][0][0]))
    assert e.node_set(0, 2, 16) == 0                                            # node reloaded: rows full again
    assert e.rows(0) == [(100, 16), (100, 16)]
    assert e.pod_cancel(0, [(20, 4, 0)], [[g]], uid) == 0                       # not in the node's podsMap any more
    assert e.rows(0) == [(100, 16), (100, 16)]                                  # -> Cancel must not run
    assert e.pod_released(uid)                                                  # scheduler-level podMaps had it


def test_auto_uid_bound_again_elsewhere_then_forgotten_is_unknown():
    """A pod with a library-assigned uid U won node 0 in a batch; then Bind puts U on node 1 as well (podMaps[U] is set
    again without a check, scheduler.go:224).  ForgetPod on node 1 deletes U from podMaps (scheduler.go:261-264), so
    U is no longer known, while node 0's podsMap still holds it and a ForgetPod there cancels node 0's rows."""
    eg = egs()
    U = 0x8000000000000000
    req = [(20, 4, 0)]
    c_off = np.array([0, 1], np.int32)
    cl = Cluster(0, [(2, 16, ([60, 100], [10, 16])), (2, 16, None)])         # node 0 the fuller: binpack picks it
    e, o = cl.handle(), cl.oracle()
    got = e.schedule_batch(c_off, np.array(req, np.int32), mode=eg.capi.EGS_MODE_ROUNDS)   # uids == NULL: U
    ref = o.schedule_batch(c_off, np.array(req, np.int64), uids=np.array([U], np.uint64))
    assert got["node"][0] == ref["node"][0] == 0 and got["status"][0] == ref["status"][0] == 0
    assert list(e.filter([1], req)) == list(o.filter([1], req)) == [1]
    st, alloc = e.bind(1, req, U)
    assert (st, alloc) == o.bind(1, req, U) and st == 0
    assert e.pod_cancel(1, req, alloc, U) == o.forget_pod(1, req, alloc, U) == 0
    assert not o.known_pod(U) and not e.pod_known(U)
    assert o.released_pod(U) and e.pod_released(U)
    assert e.rows(0) == o.rows(0) and e.rows(1) == o.rows(1)
    g = int(np.log2(got["alloc_mask"][0][0]))
    assert e.pod_cancel(0, req, [[g]], U) == o.forget_pod(0, req, [[g]], U) == 0
    assert e.rows(0) == o.rows(0) == [(60, 10), (100, 16)] and e.rows(1) == o.rows(1)
    e.close()


def test_accounting_verbs_take_pods_with_up_to_8_containers():
    """A pod with sidecars (6 containers: 4 without GPU request = {-1,-1} sentinel units, gpu.go:9-13 / allocate.go:41-45)
    that ANOTHER scheduler placed must be subtracted from the node cache exactly like the reference does (AddPod,
    replay at node load, ForgetPod, the bulk mutation stream) even though this library's filter / score / bind stop at
    4 containers -- otherwise a restarted scheduler would over-commit the node."""
    eg = egs(); cap = eg.capi
    req = [(-1, -1, 0), (30, 4, 0), (-1, -1, 0), (0, 0, 2), (-1, -1, 0), (20, 2, 0)]
    alloc = [[0], [1], [1], [2, 3], [3], [1]]
    o = oc.OracleC(0)
    o.add_node(400, 64)
    e = eg.Egs(0, 2)
    assert e.node_set_allocatable(0, 400, 64) == 0
    # AddPod
    assert e.pod_apply(0, req, alloc, 41) == 0
    o.add_pod(0, req, alloc, 41)
    assert e.rows(0) == o.rows(0) and e.pod_known(41)
    # ForgetPod gives everything back (Cancel is unchecked, gpu.go:177-191)
    assert e.pod_cancel(0, req, alloc, 41) == 0
    o.forget_pod(0, req, alloc, 41)
    assert e.rows(0) == o.rows(0) and e.pod_released(41)
    # the same through the bulk mutation stream, incl. an 8-container pod
    req8 = req + [(10, 1, 0), (-1, -1, 0)]
    alloc8 = alloc + [[0], [0]]
    assert e.mutations_apply([(cap.EGS_MUT_REPLAY, 0, req, alloc, 51), (cap.EGS_MUT_ADD, 0, req8, alloc8, 52),
                              (cap.EGS_MUT_FORGET, 0, req, alloc, 51)]) == 0
    o.add_pod(0, req, alloc, 51); o.add_pod(0, req8, alloc8, 52); o.forget_pod(0, req, alloc, 51)
    assert e.rows(0) == o.rows(0)
    # 9 containers: refused loudly, nothing applied; filter with 6 containers: refused (device path enumerates <= 4)
    before = e.rows(0)
    assert e.pod_apply(0, req8 + [(5, 1, 0)], alloc8 + [[0]], 60) == cap.EGS_ERR_BAD_ARG
    assert e.rows(0) == before
    with pytest.raises(cap.EgsError):
        e.filter([0], req)
