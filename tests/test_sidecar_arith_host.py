"""The Trade of a sidecar handle (pods of 5..8 containers, csrc/egs_device.cuh at geometry (8, 8)), compiled for the
host (csrc/host_test/device_on_host.cu) and checked against the C oracle's Trade WITHOUT a GPU:
  - egsdh_trade8c: the one-thread DFS to depth 8 that k_pass / k_gather_* run for shapes with a small leaf space;
  - egsdh_trade_split: the leaf-split reduction of k_trade_leaves + k_trade_commit -- chunks in shuffled order, chunk
    sizes that do not divide the leaf space, pruning of infeasible prefixes -- for shapes with a large one.
Score, found and all 8 masks must equal the oracle's, under both policies, on nodes of 1..8 GPUs up to the guards."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import assume, given, settings, strategies as st

import oracle_c

PAD = -(1 << 31)
W = 8
MAX_CORE, MAX_MEM = 1 << 20, 1 << 25
SENT = (-1, -1, 0)


@pytest.fixture(scope="module")
def DH():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_devhost())
    vp = C.c_void_p
    L.egsdh_trade8c.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, vp]
    L.egsdh_trade_split.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, C.c_uint64, vp, vp, vp]
    L.egsdh_leaf_eval_both.argtypes = [vp, vp, C.c_int, C.c_int, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, vp]
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


def _lists(mk, n):
    """All 8 planes of a packed word: the first n are the containers' GPU lists, the rest must be empty."""
    planes = [[g for g in range(W) if (mk >> (W * c + g)) & 1] for c in range(8)]
    assert not any(planes[n:]), f"masks beyond container {n}: {hex(mk)}"
    return planes[:n]


def _bits(g):
    return 0 if g <= 1 else 1 if g <= 2 else 2 if g <= 4 else 3


def _oracle(rows, mt, req, policy):
    o = oracle_c.OracleC(policy)
    n = o.add_node(100 * len(rows), mt * len(rows))
    o.set_rows(n, [c for c, _ in rows], [m for _, m in rows])
    return o.trade(n, req)


def _dfs(DH, rows, mt, req, policy, path):
    core, mem = _pad(rows)
    sc, mk = C.c_int32(0), C.c_uint64(0)
    if not DH.egsdh_trade8c(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data, policy, path,
                            C.byref(sc), C.byref(mk)):
        return None
    return _lists(mk.value, len(req)), sc.value


def _split(DH, rows, mt, req, policy, bits, chunk, seed):
    core, mem = _pad(rows)
    sc, mk, ev = C.c_int32(0), C.c_uint64(0), C.c_int64(0)
    ok = DH.egsdh_trade_split(core.ctypes.data, mem.ctypes.data, mt, len(req), _units(req).ctypes.data, policy, bits,
                              chunk, seed, C.byref(sc), C.byref(mk), C.byref(ev))
    return (None if not ok else (_lists(mk.value, len(req)), sc.value)), ev.value


def _n_branch(req):
    return sum(1 for u in req if u[2] == 0)


unit = st.one_of(
    st.tuples(st.integers(0, 100), st.integers(0, 40), st.just(0)).filter(lambda u: u[0] or u[1]),
    st.tuples(st.just(0), st.just(0), st.integers(1, 4)),
    st.just(SENT),
)
rows_s = st.lists(st.tuples(st.sampled_from([100, 100, 0, 37, 101]) | st.integers(0, 101), st.integers(0, 41)),
                  min_size=1, max_size=8)


@settings(max_examples=300, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=5, max_size=8), policy=st.integers(0, 1), mt=st.integers(1, 40))
def test_dfs_to_depth_8_equals_oracle(DH, rows, req, policy, mt):
    """The one-thread DFS at (8, 8), through the kernels' dispatch (for C >= 5 always the DFS), on leaf spaces up to
    2^15."""
    assume(_bits(len(rows)) * _n_branch(req) <= 15)
    assert _dfs(DH, rows, mt, req, policy, 0) == _oracle(rows, mt, req, policy)


@settings(max_examples=300, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=1, max_size=4), policy=st.integers(0, 1), mt=st.integers(1, 40),
       wider=st.booleans())
def test_both_leaf_evaluations_agree_on_every_leaf(DH, rows, req, policy, mt, wider):
    """The resolver's leaf evaluation (Req, 32-bit masks) and the leaf-split one (ReqW, 64-bit masks) are two
    definitions of the same rule: on pods of up to 4 containers they give the same score and masks for every leaf."""
    bits = 3 if wider else _bits(len(rows))
    core, mem = _pad(rows)
    u = _units(req)
    s4, m4, s8, m8 = C.c_int32(0), C.c_uint32(0), C.c_int32(0), C.c_uint64(0)
    for leaf in range(1 << (bits * _n_branch(req))):
        DH.egsdh_leaf_eval_both(core.ctypes.data, mem.ctypes.data, mt, len(req), u.ctypes.data, policy, bits, leaf,
                                C.byref(s4), C.byref(m4), C.byref(s8), C.byref(m8))
        assert (s4.value, m4.value) == (s8.value, m8.value), f"leaf {leaf}"


@settings(max_examples=300, deadline=None)
@given(rows=rows_s, req=st.lists(unit, min_size=5, max_size=8), policy=st.integers(0, 1), mt=st.integers(1, 40),
       wider=st.booleans(), chunk=st.sampled_from([1, 3, 7, 64, 100, 1000]), seed=st.integers(0, 2**63))
def test_split_reduction_equals_oracle(DH, rows, req, policy, mt, wider, chunk, seed):
    """Chunks in shuffled order, of sizes that need not divide the leaf space, with pruning; digits of the node's own
    width or of a handle's wider one (digits naming absent GPUs meet PAD and are pruned)."""
    bits = 3 if wider else _bits(len(rows))
    assume(bits * _n_branch(req) <= 15)
    got, _ = _split(DH, rows, mt, req, policy, bits, chunk, seed)
    assert got == _oracle(rows, mt, req, policy)


@settings(max_examples=150, deadline=None)
@given(g=st.integers(1, 8), mt=st.sampled_from([1, 81920, MAX_MEM]), data=st.data(), policy=st.integers(0, 1),
       chunk=st.sampled_from([5, 64, 333]), seed=st.integers(0, 2**63))
def test_split_up_to_the_guard(DH, g, mt, data, policy, chunk, seed):
    """Rows and requests up to the 2^20 / 2^25 guards, with sentinels adding +1 on top: key = score << 32 | leaf + 1
    keeps the score below 2^31."""
    gpu = st.one_of(st.just((100, mt)),
                    st.tuples(st.sampled_from([0, 1, MAX_CORE]) | st.integers(0, MAX_CORE),
                              st.sampled_from([0, MAX_MEM]) | st.integers(0, MAX_MEM)))
    rows = data.draw(st.lists(gpu, min_size=g, max_size=g))
    req = data.draw(st.lists(st.one_of(
        st.tuples(st.integers(0, MAX_CORE), st.integers(0, MAX_MEM), st.just(0)).filter(lambda u: u[0] or u[1]),
        st.tuples(st.just(0), st.just(0), st.integers(1, 3)), st.just(SENT)), min_size=5, max_size=8))
    assume(_bits(g) * _n_branch(req) <= 15)
    want = _oracle(rows, mt, req, policy)
    assert _split(DH, rows, mt, req, policy, _bits(g), chunk, seed)[0] == want
    assert _dfs(DH, rows, mt, req, policy, 1) == want


@pytest.mark.parametrize("policy", [0, 1])
def test_last_maximal_leaf_wins(DH, policy):
    """Eight equal GPUs and five sentinels: every leaf ties, and the last one -- every container on GPU 7 -- wins."""
    rows, req = [(100, 32)] * 8, [SENT] * 5
    want = _oracle(rows, 32, req, policy)
    assert want[0] == [[7]] * 5
    assert _split(DH, rows, 32, req, policy, 3, 64, 1)[0] == want
    assert _dfs(DH, rows, 32, req, policy, 1) == want


def test_sentinel_makes_a_free_gpu_not_free(DH):
    """A sentinel's +1 on a free GPU makes it non-free for a whole-GPU container after it: order matters."""
    rows = [(100, 32), (100, 32), (40, 8)]
    req = [SENT, (0, 0, 2), (0, 0, 1), SENT, SENT]
    want = _oracle(rows, 32, req, 0)
    for bits in (2, 3):
        assert _split(DH, rows, 32, req, 0, bits, 7, 3)[0] == want
    assert _dfs(DH, rows, 32, req, 0, 1) == want


def test_pruning_skips_infeasible_prefixes(DH):
    """A first container that fits one GPU only: the reduction evaluates a small part of the 2^24 leaves."""
    rows = [(100, 32)] + [(0, 0)] * 7
    req = [(60, 20, 0)] + [SENT] * 7
    got, ev = _split(DH, rows, 32, req, 0, 3, 64, 9)
    assert got == _oracle(rows, 32, req, 0)
    assert ev < (1 << 22)


@pytest.mark.parametrize("policy,rows,req", [
    (0, [(100, 32)] * 8, [(10, 4, 0)] + [SENT] * 7),
    (1, [(100, 32), (37, 9), (100, 32), (0, 0), (55, 30), (100, 32), (3, 1), (100, 32)], [SENT] * 8),
    (0, [(101, 41), (0, 0), (37, 9), (100, 32), (99, 31), (1, 1), (100, 32), (60, 2)], [(30, 8, 0), SENT, (20, 20, 0)] + [SENT] * 5),
])
def test_full_2_24_leaves(DH, policy, rows, req):
    """Eight branching containers on an 8-GPU node: the whole 2^24-leaf space, chunk size 64 as on the GPU."""
    want = _oracle(rows, 32, req, policy)
    got, ev = _split(DH, rows, 32, req, policy, 3, 64, 12345)
    assert got == want
    assert _dfs(DH, rows, 32, req, policy, 1) == want
