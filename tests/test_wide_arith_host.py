"""The 16-wide instantiation of the kernels' integer arithmetic (csrc/egs_device.cuh at G = 16: the Trade fast path
with its q*16+g key, the general DFS Trade with u16 masks, Transact and the AddPod / ForgetPod row update with index
lists of up to 16 GPUs), compiled for the host (csrc/host_test/device_on_host.cu, egsdh_*16) and checked against the
C oracle and the Python oracle WITHOUT a GPU, on nodes of 9..16 GPUs whose absent GPUs hold PAD."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import egs_oracle as po
import oracle_c

PAD = -(1 << 31)
W = 16
MAX_CORE, MAX_MEM = 1 << 20, 1 << 25


@pytest.fixture(scope="module")
def DH():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_devhost())
    L.egsdh_trade16.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.egsdh_transact16.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64]
    L.egsdh_apply16.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    return L


def _pad(rows):
    core = np.full(W, PAD, np.int32); mem = np.full(W, PAD, np.int32)
    for g, (c, m) in enumerate(rows):
        core[g], mem[g] = c, m
    return core, mem


def _units(req):
    a = np.zeros((max(1, len(req)), 3), np.int32)
    for i, u in enumerate(req):
        a[i] = u
    return a


def _masks(alloc):
    return sum(1 << (W * c + g) for c, a in enumerate(alloc) for g in a)


def _trade(DH, rows, mt, req, policy, path):
    core, mem = _pad(rows)
    sc, mk = C.c_int32(0), C.c_uint64(0)
    if not DH.egsdh_trade16(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data, policy, path,
                            C.byref(sc), C.byref(mk)):
        return None
    return [[g for g in range(W) if (mk.value >> (W * c + g)) & 1] for c in range(len(req))], sc.value


def _oracle_c(rows, mt, req, policy):
    """egso_trade on a node of len(rows) GPUs of `mt` memory holding `rows`."""
    o = oracle_c.OracleC(policy)
    n = o.add_node(100 * len(rows), mt * len(rows))
    o.set_rows(n, [c for c, _ in rows], [m for _, m in rows])
    got = o.trade(n, req)
    return None if got is None else (got[0], got[1])


def _every_trade(DH, rows, mt, req, policy):
    """The kernels' dispatch and the general DFS both return the C oracle's option (and the Python oracle's)."""
    want = _oracle_c(rows, mt, req, policy)
    opt = po.trade([po.GPU(c, m, 100, mt) for c, m in rows], po.RATERS[policy], list(req))
    assert want == (None if opt is None else (opt.allocated, opt.score))
    assert _trade(DH, rows, mt, req, policy, 0) == want
    assert _trade(DH, rows, mt, req, policy, 1) == want
    return want


unit = st.one_of(
    st.tuples(st.integers(0, 100), st.integers(0, 40), st.just(0)).filter(lambda u: u[0] or u[1]),
    st.tuples(st.just(0), st.just(0), st.integers(1, 16)),
    st.just((-1, -1, 0)),
)
rows_s = st.lists(st.tuples(st.sampled_from([100, 100, 0, 37, 101]) | st.integers(0, 101), st.integers(0, 41)),
                  min_size=9, max_size=16)


@settings(max_examples=600, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=1, max_size=4), policy=st.integers(0, 1), mt=st.integers(1, 40))
def test_trade16_equals_oracle(DH, rows, req, policy, mt):
    _every_trade(DH, rows, mt, req, policy)


@settings(max_examples=400, deadline=None)
@given(g=st.integers(9, 16), mt=st.sampled_from([1, 81920, MAX_MEM]), data=st.data(), policy=st.integers(0, 1))
def test_trade16_up_to_the_guard(DH, g, mt, data, policy):
    """Rows and requests up to the 2^20 / 2^25 guards: the fast path's key (x >> 2)*16 + g stays below 2^28."""
    gpu = st.one_of(st.just((100, mt)),
                    st.tuples(st.sampled_from([0, 1, MAX_CORE]) | st.integers(0, MAX_CORE),
                              st.sampled_from([0, MAX_MEM]) | st.integers(0, MAX_MEM)))
    rows = data.draw(st.lists(gpu, min_size=g, max_size=g))
    req = data.draw(st.lists(st.one_of(
        st.tuples(st.integers(0, MAX_CORE), st.integers(0, MAX_MEM), st.just(0)).filter(lambda u: u[0] or u[1]),
        st.tuples(st.just(0), st.just(0), st.integers(1, 16)), st.just((-1, -1, 0))), min_size=1, max_size=4))
    _every_trade(DH, rows, mt, req, policy)


@pytest.mark.parametrize("policy", [0, 1])
def test_tie_goes_to_gpu_15(DH, policy):
    """Sixteen equal GPUs: every GPU scores the same, and the last maximal one wins (gpu.go:85)."""
    alloc, score = _every_trade(DH, [(100, 32)] * 16, 32, [(10, 4, 0)], policy)
    assert alloc == [[15]]


def test_whole_gpu_counts_take_the_lowest_free_gpus(DH):
    rows = [(100, 32)] * 16
    rows[3] = (50, 16)                                            # GPU 3 is not free
    for cnt in (1, 8, 12, 15):
        alloc, _ = _every_trade(DH, rows, 32, [(0, 0, cnt)], 0)
        assert alloc == [[g for g in range(16) if g != 3][:cnt]]
    assert _every_trade(DH, rows, 32, [(0, 0, 16)], 0) is None  # 15 free GPUs
    alloc, _ = _every_trade(DH, [(100, 32)] * 16, 32, [(0, 0, 16)], 0)
    assert alloc == [list(range(16))]
    assert _every_trade(DH, [(100, 32)] * 16, 32, [(0, 0, 17)], 0) is None


def test_sentinel_on_gpu_15_adds_one(DH):
    rows = [(0, 0)] * 15 + [(40, 8)]
    alloc, score = _every_trade(DH, rows, 32, [(-1, -1, 0)], 0)
    assert alloc == [[15]]
    core, mem = _pad(rows)
    assert DH.egsdh_transact16(core.ctypes.data, mem.ctypes.data, 32, 1, _units([(-1, -1, 0)]).ctypes.data, 1 << 15)
    assert (int(core[15]), int(mem[15])) == (41, 9)               # GPU.Add of (-1, -1), gpu.go:36-37


@settings(max_examples=400, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=1, max_size=4), mt=st.integers(1, 40),
       stale=st.lists(st.tuples(st.integers(0, 15), st.integers(0, 60), st.integers(0, 30)), max_size=4))
def test_transact16_with_stale_options(DH, rows, req, mt, stale):
    """Transact of a possibly stale option: same success / failure and the same partial Adds, no rollback."""
    g = [po.GPU(c, m, 100, mt) for c, m in rows]
    opt = po.trade(g, po.rate_binpack, list(req))
    if opt is None:
        return
    for gi, dc, dm in stale:
        if gi < len(g):
            g[gi].core_avail = max(0, g[gi].core_avail - dc); g[gi].mem_avail = max(0, g[gi].mem_avail - dm)
    core, mem = _pad([(x.core_avail, x.mem_avail) for x in g])
    ok = DH.egsdh_transact16(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data, _masks(opt.allocated))
    assert bool(ok) == po.transact(g, opt)
    assert [(int(core[i]), int(mem[i])) for i in range(len(g))] == [(x.core_avail, x.mem_avail) for x in g]
    assert (core[len(g):] == PAD).all() and (mem[len(g):] == PAD).all()


def test_transact16_failure_keeps_earlier_adds(DH):
    rows = [(100, 32)] * 12
    req = [(30, 8, 0), (0, 0, 2)]
    core, mem = _pad(rows)
    core[11] = 99                                                 # the second container's GPU 11 is no longer free
    masks = _masks([[9], [10, 11]])
    assert not DH.egsdh_transact16(core.ctypes.data, mem.ctypes.data, 32, 2, _units(req).ctypes.data, masks)
    assert (int(core[9]), int(mem[9])) == (70, 24) and (int(core[10]), int(mem[10])) == (0, 0)
    assert (int(core[11]), int(mem[11])) == (99, 32)


@st.composite
def apply_records(draw):
    """(mem_total, rows, records) on one node of 9..16 GPUs; whole-GPU containers list up to 16 indices."""
    mt = draw(st.integers(1, 40))
    rows = draw(st.lists(st.tuples(st.integers(0, 103), st.integers(0, mt + 3)), min_size=9, max_size=16))
    gpu = st.integers(0, len(rows) - 1)
    container = st.one_of(
        st.tuples(st.tuples(st.integers(0, 100), st.integers(0, 40), st.just(0)), st.lists(gpu, max_size=2)),
        st.tuples(st.tuples(st.just(0), st.just(0), st.integers(1, 16)), st.lists(gpu, max_size=16)),
        st.tuples(st.just((-1, -1, 0)), st.lists(gpu, max_size=1)),
    )
    records = draw(st.lists(st.tuples(st.booleans(), st.lists(container, min_size=1, max_size=8)), min_size=1, max_size=4))
    return mt, rows, records


def _apply(DH, core, mem, mt, req, alloc, cancel):
    n_idx = np.array([len(ix) for ix in alloc], np.int32)
    idx = np.zeros((len(alloc), W), np.int32)
    for c, ix in enumerate(alloc):
        idx[c, :len(ix)] = ix
    return DH.egsdh_apply16(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data,
                            n_idx.ctypes.data, idx.ctypes.data, int(cancel))


@settings(max_examples=500, deadline=None)
@given(case=apply_records())
def test_apply16_equals_oracle(DH, case):
    """AddPod / ForgetPod row updates (NodeAllocator.Add / Forget) with fresh uids: Transact stops at the first GPU
    that cannot take its container, Cancel puts whole GPUs back at their totals."""
    mt, rows, records = case
    s = po.Scheduler(po.POLICY_BINPACK)
    s.add_node(100 * len(rows), mt * len(rows))
    s.set_rows(0, [c for c, _ in rows], [m for _, m in rows])
    na = s.nodes[0]
    core, mem = _pad(rows)
    for uid, (cancel, containers) in enumerate(records):
        req = [u for u, _ in containers]
        alloc = [list(ix) for _, ix in containers]
        got = _apply(DH, core, mem, mt, req, alloc, cancel)
        if cancel:
            na.pods_map[uid] = True
            na.forget(req, alloc, uid)
            assert got == 1
        else:
            assert bool(got) == na.add(uid, po.GPUOption(request=req, allocated=alloc))
        assert [(int(core[g]), int(mem[g])) for g in range(len(rows))] == s.rows(0)
        assert (core[len(rows):] == PAD).all() and (mem[len(rows):] == PAD).all()


def test_add_and_cancel_a_12_gpu_container(DH):
    rows = [(100, 32)] * 16
    core, mem = _pad(rows)
    alloc = [list(range(2, 14))]
    assert _apply(DH, core, mem, 32, [(0, 0, 12)], alloc, False) == 1
    assert [int(core[g]) for g in range(16)] == [100, 100] + [0] * 12 + [100, 100]
    assert _apply(DH, core, mem, 32, [(0, 0, 12)], alloc, True) == 1
    assert [(int(core[g]), int(mem[g])) for g in range(16)] == rows
