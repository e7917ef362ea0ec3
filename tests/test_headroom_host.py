"""Headroom without a GPU.  The independence claim egs_headroom rests on -- under a stream of pods of one shape every
node binds on its own, so a dry run's binds per node are what the node's own Assume / Allocate loop makes -- is checked
on the oracle: the Python headroom model (headroom_model) equals a pod-by-pod oracle dry run of K identical pods, node
by node.  Then headroom_node, the loop k_headroom runs, compiled for the host (csrc/host_test/device_on_host.cu),
equals the model at every handle geometry up to the int32 guards."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import egs_oracle as po
import headroom_cases as hc
from headroom_model import allocator, node_headroom, oracle_headroom
from oracle_harness import Cluster, oracle_batch

SENT = hc.SENT
SHAPES = [
    [(25, 4, 0)], [(0, 4, 0)], [(50, 8, 0)], [(10, 2, 0)],          # single fractional, core 0 included
    [(0, 0, 1)], [(0, 0, 2)], [(0, 0, 8)],                          # whole GPUs
    [(20, 4, 0), (10, 2, 0)], [(30, 8, 0), (30, 8, 0), (10, 2, 0)],  # multi-container
    [(0, 0, 1), SENT], [SENT, (25, 4, 0)], [(0, 0, 1), (10, 2, 0)],  # GPU + sentinel, mixed
]


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_model_equals_oracle_dry_run(policy, seed):
    """Seeded clusters with a history (cached, stale cached and unfit options; over-totals rows): for every shape the
    model's binds and failed binds per node equal the EGS_OK and EGS_ERR_TRANSACT pods of a dry run of
    K = sum + 40 identical pods, and every pod after the last bind is EGS_ERR_NOFIT."""
    rng = np.random.default_rng([seed, policy])
    cl = Cluster(policy, hc.nodes(rng, 24))
    hist = hc.history(rng, cl.nodes, SHAPES, 60, 30)
    n_stale = n_failed = 0
    for sh in SHAPES:
        o = cl.oracle()
        c_off, units, uids, mut_at, recs = hist
        oracle_batch(o, c_off, units, uids, recs, mut_at)
        ok, failed, capped = (np.array(x) for x in oracle_headroom(o, cl.nodes, policy, sh))
        assert not capped.any()
        n_failed += int(failed.sum())
        n_stale += sum(o.peek(n, sh) is not None and o.trade(n, sh) is not None and o.peek(n, sh) != o.trade(n, sh)
                       for n in range(cl.n_nodes))
        K = int(ok.sum() + failed.sum()) + 40
        c_off, units = hc.identical(sh, K)
        out = oracle_batch(o, c_off, units, np.arange(10**6, 10**6 + K, dtype=np.uint64))
        hc.check_dry_run(ok, failed, out, what=f"shape {sh}")
    assert n_stale > 0 and n_failed > 0, "the history made no stale option that fails its Transact"


def test_model_limit_and_unbounded_shapes():
    """A {0,0} container and a pod of sentinels alone fit forever: the model stops at the limit and says so.  A
    finite shape stops exactly at a limit below its count."""
    na = allocator([(100, 16), (30, 2)], 16, 0)
    for sh in ([(0, 0, 0)], [SENT], [SENT, SENT]):
        assert node_headroom(na, sh, limit=57) == (57, 0, True)
    assert node_headroom(na, [(25, 4, 0)]) == (4, 0, False)
    assert node_headroom(na, [(25, 4, 0)], limit=3) == (3, 0, True)
    assert node_headroom(na, [(25, 4, 0)], limit=4) == (4, 0, False)
    assert node_headroom(allocator([(0, 0)], 16, 0), [(0, 0, 0)], limit=5) == (5, 0, True)
    assert node_headroom(na, [(0, 0, 2)]) == (0, 0, False)


# ------------------------------------------------------------------------------------------------ the kernel's loop
OPT_ABSENT, OPT_CACHED, OPT_UNFIT = 0, 1, 2
MAX_CORE, MAX_MEM = 1 << 20, 1 << 25


@pytest.fixture(scope="module")
def DH():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_devhost())
    L.egsdh_headroom.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                 C.c_int, C.c_uint64, C.c_int, C.c_void_p]
    return L


def _kernel_loop(DH, G, planes, rows, mt, req, policy, state, masks, limit):
    core = np.full(G, -(1 << 31), np.int32); mem = core.copy()
    for g, (c, m) in enumerate(rows):
        core[g], mem[g] = c, m
    u = np.array(req, np.int32).reshape(-1, 3)
    out = np.zeros(3, np.int32)
    DH.egsdh_headroom(G, planes, core.ctypes.data, mem.ctypes.data, mt, len(req), u.ctypes.data, policy, state, masks,
                      limit, out.ctypes.data)
    return int(out[0]), int(out[1]), bool(out[2])


@st.composite
def node_case(draw):
    """(G, planes, mem_total, rows, request, stale rows) on a handle geometry: 8 or 16 GPUs per row, 4 or 8 mask
    planes; rows anywhere up to the int32 guards or near a small total.  A request has up to 2 branching containers
    (fractional or sentinel, tried on every GPU) and whole-GPU ones, which do not branch: up to 8 containers with 8
    planes."""
    G, planes = draw(st.sampled_from([(8, 4), (16, 4), (8, 8)]))
    big = draw(st.booleans())
    mt = draw(st.sampled_from([MAX_MEM, MAX_MEM - 1, 81920])) if big else draw(st.integers(1, 40))
    hi_c, hi_m = (MAX_CORE, MAX_MEM) if big else (130, mt + 5)
    gpu = st.one_of(st.just((100, mt)), st.tuples(st.integers(0, hi_c), st.integers(0, hi_m)))
    rows = draw(st.lists(gpu, min_size=1, max_size=G))
    frac = st.tuples(st.integers(0, 100), st.integers(0, max(1, hi_m // 8)), st.just(0)).filter(lambda u: u[0] or u[1])
    branching = draw(st.lists(st.one_of(frac, st.just(SENT)), min_size=1, max_size=2))
    if planes == 4:
        whole = draw(st.lists(st.tuples(st.just(0), st.just(0), st.integers(1, 3)), max_size=1))
    else:
        whole = draw(st.lists(st.just((0, 0, 1)), min_size=5 - len(branching), max_size=8 - len(branching)))
    req = draw(st.permutations(branching + whole))
    stale = draw(st.lists(st.tuples(st.integers(0, len(rows) - 1), st.integers(-3, 60), st.integers(-3, 60)), max_size=3))
    return G, planes, mt, rows, list(req), stale


@settings(max_examples=300, deadline=None)
@given(case=node_case(), policy=st.integers(0, 1), limit=st.integers(1, 24), cached=st.booleans())
def test_kernel_loop_equals_model(DH, case, policy, limit, cached):
    """headroom_node from each option state: an entry Traded on the rows before `stale` changed them (Transacted
    first, failing where it no longer fits), no entry, and -- when Trade fails on the current rows -- the
    "known not to fit" memo."""
    G, planes, mt, rows, req, stale = case
    req = [tuple(u) for u in req]
    option = None
    if cached:
        t = po.trade([po.GPU(c, m, 100, mt) for c, m in rows], po.RATERS[policy], req)
        option = None if t is None else (t.allocated, t.score)
    rows = list(rows)
    for g, dc, dm in stale:                                      # rows changed under the cached option
        c, m = rows[g]
        rows[g] = (max(0, c - dc), max(0, m - dm))
    want = node_headroom(allocator(rows, mt, policy, req, option), req, limit)
    if option is not None:
        masks = sum(1 << (G * c + g) for c, a in enumerate(option[0]) for g in a)
        assert _kernel_loop(DH, G, planes, rows, mt, req, policy, OPT_CACHED, masks, limit) == want
    else:
        assert _kernel_loop(DH, G, planes, rows, mt, req, policy, OPT_ABSENT, 0, limit) == want
        if want[0] == 0:
            assert _kernel_loop(DH, G, planes, rows, mt, req, policy, OPT_UNFIT, 0, limit) == (0, 0, False)


@pytest.mark.parametrize("G,planes", [(8, 4), (16, 4), (8, 8)])
def test_kernel_loop_at_the_limit_bound(DH, G, planes):
    """EGS_HEADROOM_MAX_LIMIT binds of a pod of sentinels alone on a GPU at the guards beside an empty one: the rows
    grow by up to 8 per bind and the loop stops at the limit with an option left.  Then a 1-core, 1-MiB pod, of which
    the GPU at the guards holds more than the limit."""
    import egs_b200
    limit = egs_b200.capi.EGS_HEADROOM_MAX_LIMIT
    rows = [(MAX_CORE, MAX_MEM), (0, 0)]                      # two GPUs: the widest range, every sidecar on one GPU
    assert _kernel_loop(DH, G, planes, rows, MAX_MEM, [SENT] * planes, 0, OPT_ABSENT, 0, limit) == (limit, 0, True)
    assert _kernel_loop(DH, G, planes, rows, MAX_MEM, [(1, 1, 0)], 0, OPT_ABSENT, 0, limit) == (limit, 0, True)
