"""The kernels' integer arithmetic -- csrc/egs_device.cuh: the Trade fast path (prefix/suffix maxima,
unsigned-min PAD trick, packed q*8+g key) and its one-GPU-per-lane form in the resolver, the general DFS Trade,
Transact and the AddPod / ForgetPod row update -- compiled for the host
(csrc/host_test/device_on_host.cu) and checked against the oracle WITHOUT a GPU.  Same source the kernels
inline; the device SASS is unaffected by the host build."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import egs_oracle as po

PAD = -(1 << 31)


@pytest.fixture(scope="module")
def DH():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_devhost())
    L.egsdh_trade.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.egsdh_trade_leaves.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.egsdh_transact.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint32]
    L.egsdh_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    L.egsdh_trade_lanes.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.egsdh_is_single.argtypes = [C.c_int, C.c_void_p]
    for f in ("egsdh_cand_key", "egsdh_fit_term", "egsdh_score_term"):
        getattr(L, f).restype = C.c_uint64
    L.egsdh_cand_key.argtypes = [C.c_int32, C.c_uint32]
    L.egsdh_fit_term.argtypes = [C.c_uint32]
    L.egsdh_score_term.argtypes = [C.c_uint32, C.c_int32]
    return L


def _pad(rows):
    core = np.full(8, PAD, np.int32); mem = np.full(8, PAD, np.int32)
    for g, (c, m) in enumerate(rows):
        core[g], mem[g] = c, m
    return core, mem


def _units(req):
    a = np.zeros((max(1, len(req)), 3), np.int32)
    for i, u in enumerate(req):
        a[i] = u
    return a


def _trade(DH, rows, mt, req, policy, path):
    core, mem = _pad(rows)
    u = _units(req)
    sc, mk = C.c_int32(0), C.c_uint32(0)
    ok = DH.egsdh_trade(core.ctypes.data, mem.ctypes.data, mt, len(req), u.ctypes.data, policy, path, C.byref(sc), C.byref(mk))
    if not ok:
        return None
    alloc = [[g for g in range(8) if (mk.value >> (8 * c + g)) & 1] for c in range(len(req))]
    return alloc, sc.value


def _trade_lanes(DH, rows, req, policy):
    """trade_lane_key, the one-GPU-per-lane Trade of the resolver's single-container pods, maxed over the lanes."""
    core, mem = _pad(rows)
    (rq_core, rq_mem, _), = req
    sc, mk = C.c_int32(0), C.c_uint32(0)
    if not DH.egsdh_trade_lanes(core.ctypes.data, mem.ctypes.data, rq_core, rq_mem, policy, C.byref(sc), C.byref(mk)):
        return None
    return [[g for g in range(8) if (mk.value >> g) & 1]], sc.value


unit = st.one_of(
    st.tuples(st.integers(0, 100), st.integers(0, 40), st.just(0)).filter(lambda u: u[0] or u[1]),
    st.tuples(st.just(0), st.just(0), st.integers(1, 3)),
    st.just((-1, -1, 0)),
)
rows_s = st.lists(st.tuples(st.integers(0, 101), st.integers(0, 41)), min_size=1, max_size=8)


@settings(max_examples=600, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=1, max_size=4), policy=st.integers(0, 1), mt=st.integers(1, 40))
def test_kernel_trade_equals_oracle(DH, rows, req, policy, mt):
    g = [po.GPU(c, m, 100, mt) for c, m in rows]
    opt = po.trade(g, po.RATERS[policy], list(req))
    want = None if opt is None else (opt.allocated, opt.score)
    assert _trade(DH, rows, mt, req, policy, 0) == want          # the dispatch the kernels use
    assert _trade(DH, rows, mt, req, policy, 1) == want          # general DFS on every request
    if DH.egsdh_is_single(len(req), _units(req).ctypes.data):
        assert _trade_lanes(DH, rows, req, policy) == want       # the resolver's per-lane form


@settings(max_examples=800, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=1, max_size=4), policy=st.integers(0, 1), mt=st.integers(1, 40))
def test_leaf_parallel_trade_equals_oracle(DH, rows, req, policy, mt):
    """trade_leaf_eval / trade_leaf_space (the Trade the resolver spreads over the lanes of a warp, one DFS leaf per
    lane): the maximal (score, leaf index) over all leaves is the option gpu.go:65-129 returns -- same Allocated,
    same Score, same 'last maximal leaf wins', including whole-GPU and sentinel containers and 3/5/6/7-GPU nodes."""
    g = [po.GPU(c, m, 100, mt) for c, m in rows]
    opt = po.trade(g, po.RATERS[policy], list(req))
    want = None if opt is None else (opt.allocated, opt.score)
    core, mem = _pad(rows)
    u = _units(req)
    sc, mk = C.c_int32(0), C.c_uint32(0)
    ok = DH.egsdh_trade_leaves(core.ctypes.data, mem.ctypes.data, mt, len(req), u.ctypes.data, policy, C.byref(sc), C.byref(mk))
    got = None if not ok else ([[gg for gg in range(8) if (mk.value >> (8 * c + gg)) & 1] for c in range(len(req))], sc.value)
    assert got == want


@settings(max_examples=600, deadline=None)
@given(rows=st.lists(st.tuples(st.integers(0, 100), st.sampled_from([0, 1, 1024, 40960, 81920, (1 << 25)])), min_size=1, max_size=8),
       core=st.integers(0, 99), mem=st.sampled_from([0, 1, 1024, 4096, 40960, 81920, (1 << 25) - 7]), policy=st.integers(0, 1))
def test_fast_path_single_container_large_values(DH, rows, core, mem, policy):
    """The fast path with realistic magnitudes (MB-scale memory up to the 2^25 guard): no int32 overflow,
    score == Range/2*100, last maximal GPU wins."""
    if core == 0 and mem == 0:
        mem = 1
    mt = 1 << 25
    req = [(core, mem, 0)]
    g = [po.GPU(c, m, 100, mt) for c, m in rows]
    opt = po.trade(g, po.RATERS[policy], req)
    want = None if opt is None else (opt.allocated, opt.score)
    u = _units(req)
    assert DH.egsdh_is_single(1, u.ctypes.data) == 1
    assert _trade(DH, rows, mt, req, policy, 0) == want
    assert _trade_lanes(DH, rows, req, policy) == want


@settings(max_examples=400, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=1, max_size=4), mt=st.integers(1, 40), stale=st.lists(st.tuples(st.integers(0, 7), st.integers(0, 60), st.integers(0, 30)), max_size=3))
def test_kernel_transact_equals_oracle(DH, rows, req, mt, stale):
    """Transact with a possibly STALE option (rows changed after the option was made): same success/failure,
    same partial application without rollback (gpu.go:153-175)."""
    g = [po.GPU(c, m, 100, mt) for c, m in rows]
    opt = po.trade(g, po.rate_binpack, list(req))
    if opt is None:
        return
    for gi, dc, dm in stale:                                      # somebody else consumed resources meanwhile
        if gi < len(g):
            g[gi].core_avail = max(0, g[gi].core_avail - dc); g[gi].mem_avail = max(0, g[gi].mem_avail - dm)
    core, mem = _pad([(x.core_avail, x.mem_avail) for x in g])
    masks = 0
    for c, a in enumerate(opt.allocated):
        for gi in a:
            masks |= 1 << (8 * c + gi)
    ok = DH.egsdh_transact(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data, masks)
    assert bool(ok) == po.transact(g, opt)
    assert [(int(core[i]), int(mem[i])) for i in range(len(g))] == [(x.core_avail, x.mem_avail) for x in g]


@st.composite
def apply_records(draw):
    """(mem_total, rows, records) on one node of 1..8 GPUs whose rows may sit above their totals.  A record is
    (cancel, [(unit, GPU indices)]) with up to 8 fractional, whole-GPU or sentinel containers; the index lists are
    what the annotations hold, so they may repeat a GPU or name one that no longer fits."""
    mt = draw(st.integers(1, 40))
    rows = draw(st.lists(st.tuples(st.integers(0, 103), st.integers(0, mt + 3)), min_size=1, max_size=8))
    gpu = st.integers(0, len(rows) - 1)
    container = st.one_of(
        st.tuples(st.tuples(st.integers(0, 100), st.integers(0, 40), st.just(0)), st.lists(gpu, max_size=2)),
        st.tuples(st.tuples(st.just(0), st.just(0), st.integers(1, 3)), st.lists(gpu, max_size=4)),
        st.tuples(st.just((-1, -1, 0)), st.lists(gpu, max_size=1)),
    )
    records = draw(st.lists(st.tuples(st.booleans(), st.lists(container, min_size=1, max_size=8)), min_size=1, max_size=4))
    return mt, rows, records


@settings(max_examples=600, deadline=None)
@given(case=apply_records())
def test_apply_row_update_equals_oracle(DH, case):
    """apply_op, the row update of k_apply and k_apply_many, against the oracle's NodeAllocator.Add / Forget (what
    AddPod / ForgetPod call) with fresh uids, so every record reaches the rows: Transact stops at the first GPU that
    cannot take its container and keeps the Adds before it; Cancel puts a whole-GPU container's GPUs back at their
    totals; a fractional container uses its first index only."""
    mt, rows, records = case
    s = po.Scheduler(po.POLICY_BINPACK)
    s.add_node(100 * len(rows), mt * len(rows))
    s.set_rows(0, [c for c, _ in rows], [m for _, m in rows])
    na = s.nodes[0]
    core, mem = _pad(rows)
    for uid, (cancel, containers) in enumerate(records):
        req = [u for u, _ in containers]
        alloc = [list(ix) for _, ix in containers]
        n_idx = np.array([len(ix) for ix in alloc], np.int32)
        idx = np.zeros((len(alloc), 8), np.int32)
        for c, ix in enumerate(alloc):
            idx[c, :len(ix)] = ix
        got = DH.egsdh_apply(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data,
                             n_idx.ctypes.data, idx.ctypes.data, int(cancel))
        if cancel:
            na.pods_map[uid] = True                                   # the pod is on the node: Forget cancels it
            na.forget(req, alloc, uid)
            assert got == 1
        else:
            assert bool(got) == na.add(uid, po.GPUOption(request=req, allocated=alloc))
        assert [(int(core[g]), int(mem[g])) for g in range(len(rows))] == s.rows(0)
        assert (core[len(rows):] == PAD).all() and (mem[len(rows):] == PAD).all()


def _trade_leaves(DH, rows, mt, req, policy):
    core, mem = _pad(rows)
    u = _units(req)
    sc, mk = C.c_int32(0), C.c_uint32(0)
    if not DH.egsdh_trade_leaves(core.ctypes.data, mem.ctypes.data, mt, len(req), u.ctypes.data, policy, C.byref(sc), C.byref(mk)):
        return None
    return [[g for g in range(8) if (mk.value >> (8 * c + g)) & 1] for c in range(len(req))], sc.value


def _every_trade_equals_oracle(DH, rows, mt, req, policy):
    """The kernels' dispatch, the general DFS, the leaf-parallel Trade and (single-container shapes) the per-lane
    form all return the oracle's option.  Returns it."""
    g = [po.GPU(c, m, 100, mt) for c, m in rows]
    opt = po.trade(g, po.RATERS[policy], list(req))
    want = None if opt is None else (opt.allocated, opt.score)
    assert _trade(DH, rows, mt, req, policy, 0) == want
    assert _trade(DH, rows, mt, req, policy, 1) == want
    assert _trade_leaves(DH, rows, mt, req, policy) == want
    if DH.egsdh_is_single(len(req), _units(req).ctypes.data):
        assert _trade_lanes(DH, rows, req, policy) == want
    return want


# ---- the int32 guard (DESIGN §1): free core <= 2^20 and free memory <= 2^25 per GPU, requests within the same
# bounds.  The score comes closest to 2^31 with k = 0 (no container holds exactly one GPU: whole-GPU containers of
# count >= 2 only): Range/1*100 with Range up to (2^25 + 2^20) / 2, about 1.73e9.
MAX_CORE, MAX_MEM = 1 << 20, 1 << 25


@st.composite
def guard_rows(draw):
    """(mem_total, rows): GPUs free at their totals (whole-GPU containers can take them), just above them, or
    anywhere up to the guard."""
    mt = draw(st.sampled_from([1, 81920, MAX_MEM - 1, MAX_MEM]))
    gpu = st.one_of(
        st.just((100, mt)),
        st.tuples(st.integers(100, 103), st.integers(mt, mt + 3)).map(lambda r: (r[0], min(r[1], MAX_MEM))),
        st.tuples(st.one_of(st.integers(0, MAX_CORE), st.sampled_from([0, MAX_CORE - 1, MAX_CORE])),
                  st.one_of(st.integers(0, MAX_MEM), st.sampled_from([0, MAX_MEM - 1, MAX_MEM]))),
    )
    return mt, draw(st.lists(gpu, min_size=1, max_size=8))


guard_unit = st.one_of(
    st.tuples(st.one_of(st.integers(0, MAX_CORE), st.sampled_from([0, 1, 100, MAX_CORE])),
              st.one_of(st.integers(0, MAX_MEM), st.sampled_from([0, 1, MAX_MEM])), st.just(0)).filter(lambda u: u[0] or u[1]),
    st.tuples(st.just(0), st.just(0), st.integers(1, 3)),
    st.just((-1, -1, 0)),
)
k0_req = st.lists(st.tuples(st.just(0), st.just(0), st.integers(2, 4)), min_size=1, max_size=2)


@settings(max_examples=800, deadline=None)
@given(mrows=guard_rows(), req=st.one_of(st.lists(guard_unit, min_size=1, max_size=4), k0_req), policy=st.integers(0, 1))
def test_every_trade_at_the_int32_guard(DH, mrows, req, policy):
    """Rows and requests up to the guard, whole-GPU containers on GPUs at, above and far from their totals, k = 0
    shapes: every Trade the kernels run equals the oracle's (which computes in int64)."""
    mt, rows = mrows
    _every_trade_equals_oracle(DH, rows, mt, req, policy)


@pytest.mark.parametrize("policy", [0, 1])
def test_k0_score_near_the_int32_limit(DH, policy):
    """The largest score the guard admits: the free GPUs taken by whole-GPU containers of count 2, the last GPU at
    (2^20, 2^25)."""
    for req in ([(0, 0, 2)], [(0, 0, 2), (0, 0, 2)]):
        n = 2 * len(req)
        rows = [(100, MAX_MEM)] * n + [(MAX_CORE, MAX_MEM)]
        alloc, score = _every_trade_equals_oracle(DH, rows, MAX_MEM, req, policy)
        assert sorted(sum(alloc, [])) == list(range(n))
        assert score == (0 if policy else (MAX_MEM + MAX_CORE) // 2 * 100) and score < 2**31


@settings(max_examples=600, deadline=None)
@given(rows=st.lists(st.tuples(st.integers(97, 103), st.integers(13, 19)), min_size=1, max_size=8),
       req=st.lists(st.one_of(st.tuples(st.integers(0, 3), st.integers(0, 3), st.just(0)).filter(lambda u: u[0] or u[1]),
                              st.tuples(st.just(0), st.just(0), st.integers(1, 3)), st.just((-1, -1, 0))),
                    min_size=1, max_size=4),
       policy=st.integers(0, 1))
def test_whole_gpu_trade_above_totals(DH, rows, req, policy):
    """GPUs of 16 MiB around their totals (97..103 core, 13..19 MiB): only a GPU at exactly (100, 16) is free for a
    whole-GPU container, also after the shape's own fractional and sidecar containers moved it there; Transact of the
    resulting option agrees too."""
    want = _every_trade_equals_oracle(DH, rows, 16, req, policy)
    if want is None:
        return
    g = [po.GPU(c, m, 100, 16) for c, m in rows]
    ok = po.transact(g, po.GPUOption(request=list(req), allocated=want[0], score=want[1]))
    core, mem = _pad(rows)
    masks = sum(1 << (8 * c + gi) for c, a in enumerate(want[0]) for gi in a)
    assert bool(DH.egsdh_transact(core.ctypes.data, mem.ctypes.data, 16, len(req), _units(req).ctypes.data, masks)) == ok
    assert [(int(core[i]), int(mem[i])) for i in range(len(g))] == [(x.core_avail, x.mem_avail) for x in g]


def test_keys_and_digest_terms(DH):
    for node, score in [(0, 0), (5, 600), (99999, 2050500), (2**31 - 1, 0)]:
        assert DH.egsdh_fit_term(node) == po.fit_digest_term(node)
        assert DH.egsdh_score_term(node, score) == po.score_digest_term(node, score)
    # ordering: higher score first, then LOWER node id
    k = DH.egsdh_cand_key
    assert k(600, 7) > k(500, 0) and k(600, 3) > k(600, 4) and k(0, 0) > 0
