"""The eviction what-if without a GPU: evict_node, the per-node answer k_evict runs, compiled for the host
(csrc/host_test/device_on_host.cu), equals the model on the Python oracle (evict_model: Forget of each victim, then
Assume / Score / Allocate on a copy of the node) at every handle geometry and under both policies.

A node's case: rows (free, partly used, empty, above their totals, or at the guards); a pending pod; the node's cached
option of it, Traded before later pods changed the rows (so it may be stale), or none; the uids of the node's podsMap
with the placements they hold; and a victim list drawn from those pods, unknown uids and repeats.  The kernel gets the
option entry's state and the victims that apply, as egs_evict_fit hands them over."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import egs_oracle as po
from evict_model import applied, node_evict
from headroom_model import allocator

SENT = (-1, -1, 0)
OPT_ABSENT, OPT_CACHED, OPT_UNFIT = 0, 1, 2
MAX_CORE, MAX_MEM = 1 << 20, 1 << 25
GEOMETRIES = [(8, 4), (16, 4), (8, 8)]


@pytest.fixture(scope="module")
def DH():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_devhost())
    vp, i = C.c_void_p, C.c_int
    L.egsdh_evict.argtypes = [i, i, vp, vp, i, i, vp, i, i, i, vp, i, vp, vp]
    return L


def pack(alloc, G):
    return sum(1 << (G * c + g) for c, a in enumerate(alloc or []) for g in (a or []))


# ------------------------------------------------------------------------------------------------ cases
class RngPick:
    def __init__(self, rng):
        self.r = rng

    def int(self, lo, hi):
        return int(self.r.integers(lo, hi + 1))


class DrawPick:
    def __init__(self, draw):
        self.d = draw

    def int(self, lo, hi):
        return self.d(st.integers(lo, hi))


def gen_case(p, G, planes):
    """(mem_total, rows, req, option, pods, victims).  pods: {uid: (units, alloc)} of the node's podsMap; the ones
    placed after the option was Traded changed the rows under it.  victims: [(units, alloc, uid)]."""
    mt = (16, 40, 81920, MAX_MEM)[p.int(0, 3)]
    g = p.int(1, G)
    rows = []
    for _ in range(g):
        k = p.int(0, 4)
        if k == 0:
            rows.append((100, mt))
        elif k == 1:
            rows.append((p.int(0, 100), p.int(0, mt)))
        elif k == 2:                                          # above the totals
            rows.append((p.int(101, 140), min(MAX_MEM, mt + p.int(1, mt // 4 + 3))))
        elif k == 3:
            rows.append((0, 0))
        else:                                                 # at the guards
            rows.append((MAX_CORE - p.int(0, 3), MAX_MEM - p.int(0, 3)))

    def frac():                                               # memory small enough that no cancel leaves int32
        u = (p.int(0, 100), p.int(0, min(mt // 2, 1 << 16)), 0)
        return u if u[0] or u[1] else (1, 0, 0)

    def pod(n_max):
        """A placed pod on this node: units and GPU lists (a fractional or sentinel container on one GPU, sometimes
        on none; a whole-GPU container on up to 8 distinct GPUs)."""
        units, alloc = [], []
        for _ in range(p.int(1, n_max)):
            k = p.int(0, 3)
            if k == 0:
                n = p.int(1, min(8, g))
                gpus = sorted({p.int(0, g - 1) for _ in range(n)})
                units.append((0, 0, len(gpus))); alloc.append(gpus)
            else:
                units.append(SENT if k == 1 else frac())
                alloc.append([] if p.int(0, 9) == 0 else [p.int(0, g - 1)])
        return units, alloc

    branching = [SENT if p.int(0, 3) == 0 else frac() for _ in range(p.int(1, 2))]
    whole = [(0, 0, p.int(1, 2)) for _ in range(p.int(0, planes - len(branching)))]
    req = branching + whole
    for k in range(len(req) - 1, 0, -1):                       # shuffle
        j = p.int(0, k)
        req[k], req[j] = req[j], req[k]
    option = None
    if p.int(0, 1):
        t = po.trade([po.GPU(c, m, 100, mt) for c, m in rows], po.RATERS[0 if p.int(0, 1) else 1], req)
        option = None if t is None else (t.allocated, t.score)
    pods = {}
    for uid in range(1, p.int(1, 5) + 1):                      # pods already in the rows, then pods placed later
        pods[uid] = pod(3)
    gpus = [po.GPU(c, m, 100, mt) for c, m in rows]
    for uid in range(10, 10 + p.int(0, 3)):
        units, alloc = pods[uid] = pod(2)
        po.transact(gpus, po.GPUOption(request=units, allocated=alloc))   # AddPod: stops at the first GPU it misses
    rows = [(x.core_avail, x.mem_avail) for x in gpus]
    victims = []
    for _ in range(p.int(0, 6)):
        k = p.int(0, 5)
        if k == 0:                                             # a uid the node's podsMap does not hold
            units, alloc = pod(2)
            victims.append((units, alloc, 100 + p.int(0, 3)))
        else:
            uid = sorted(pods)[p.int(0, len(pods) - 1)]
            victims.append(pods[uid] + (uid,))
    freed = [po.GPU(c, m, 100, mt) for c, m in rows]
    for units, alloc, _ in applied(pods, victims):
        po.cancel(freed, po.GPUOption(request=units, allocated=alloc))
    if any(x.core_avail < 0 or x.mem_avail < 0 for x in freed):
        victims = []                                           # a sentinel taken back off a GPU at 0: rows stay >= 0
    return mt, rows, req, option, pods, victims


def model_answer(G, mt, rows, req, policy, option, pods, victims):
    na = allocator(rows, mt, policy, req, option)
    na.pods_map = {uid: True for uid in pods}
    st_, score, alloc = node_evict(na, req, victims)
    return st_, score, pack(alloc, G)


def kernel_answer(DH, G, planes, mt, rows, req, policy, state, option, victims):
    import egs_b200
    core = np.full(G, -(1 << 31), np.int32); mem = core.copy()
    for g, (c, m) in enumerate(rows):
        core[g], mem[g] = c, m
    u = np.array(req, np.int32).reshape(-1, 3)
    mk = np.array([pack(option[0], G) if option else 0], np.uint64)
    recs = egs_b200.capi.mutations_array([(1, 0, units, alloc, uid) for units, alloc, uid in victims])
    out = np.zeros(2, np.int32)
    DH.egsdh_evict(G, planes, core.ctypes.data, mem.ctypes.data, mt, len(req), u.ctypes.data, policy, state,
                   option[1] if option else 0, mk.ctypes.data, len(victims), recs.ctypes.data, out.ctypes.data)
    return int(out[0]), int(out[1]), int(mk[0])


def check(DH, G, planes, case, policy):
    """The kernel's answer from every option state the library can hold equals the model.  Returns the model's answer
    and the victims that apply."""
    mt, rows, req, option, pods, victims = case
    want = model_answer(G, mt, rows, req, policy, option, pods, victims)
    app = applied(pods, victims)
    if option is not None:
        assert kernel_answer(DH, G, planes, mt, rows, req, policy, OPT_CACHED, option, app) == want
    else:
        assert kernel_answer(DH, G, planes, mt, rows, req, policy, OPT_ABSENT, None, app) == want
        if po.trade([po.GPU(c, m, 100, mt) for c, m in rows], po.RATERS[policy], req) is None:
            # the "known not to fit" memo is taken on these rows: it holds until a victim applies
            assert kernel_answer(DH, G, planes, mt, rows, req, policy, OPT_UNFIT, None, app) == want
    return want, app


# ------------------------------------------------------------------------------------------------ seeded
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("G,planes", GEOMETRIES)
def test_kernel_equals_model_seeded(DH, G, planes, policy):
    """600 seeded nodes per geometry and policy; every kind of case the definition distinguishes occurs."""
    rng = np.random.default_rng([G, planes, policy])
    seen = dict(ok=0, nofit=0, stale_fails=0, stale_fixed_by_victims=0, unfit_freed=0, unfit_kept=0,
                whole_victim=0, sentinel_victim=0, above_totals=0, duplicate=0)
    for _ in range(600):
        case = gen_case(RngPick(rng), G, planes)
        mt, rows, req, option, pods, victims = case
        (status, _, _), app = check(DH, G, planes, case, policy)
        seen["ok"] += status == po.EGS_OK
        seen["nofit"] += status == po.EGS_ERR_NOFIT
        if option is not None:
            seen["stale_fails"] += status == po.EGS_ERR_TRANSACT
            alone = model_answer(G, mt, rows, req, policy, option, pods, [])
            seen["stale_fixed_by_victims"] += alone[0] == po.EGS_ERR_TRANSACT and status == po.EGS_OK
        elif po.trade([po.GPU(c, m, 100, mt) for c, m in rows], po.RATERS[policy], req) is None:
            seen["unfit_freed"] += bool(app) and status == po.EGS_OK
            seen["unfit_kept"] += not app
        seen["whole_victim"] += any(u[2] > 0 for v in app for u in v[0])
        seen["sentinel_victim"] += any(tuple(u) == SENT for v in app for u in v[0])
        seen["above_totals"] += any(c > 100 or m > mt for c, m in rows)
        seen["duplicate"] += len(app) < len([v for v in victims if v[2] in pods])
    assert all(seen.values()), seen


# ------------------------------------------------------------------------------------------------ hypothesis
@st.composite
def node_case(draw):
    G, planes = draw(st.sampled_from(GEOMETRIES))
    return G, planes, gen_case(DrawPick(draw), G, planes)


@settings(max_examples=300, deadline=None)
@given(case=node_case(), policy=st.integers(0, 1))
def test_kernel_equals_model(DH, case, policy):
    G, planes, c = case
    check(DH, G, planes, c, policy)


# ------------------------------------------------------------------------------------------------ named cases
@pytest.mark.parametrize("G,planes", GEOMETRIES)
def test_named_cases(DH, G, planes):
    """Hand-made nodes for each rule of the definition."""
    mt = 40
    frac = [(50, 20, 0)]
    # a stale cached option on GPU 0: it fails while pod 7 holds the GPU, and succeeds once pod 7 goes
    rows = [(30, 10), (100, 40)]
    option = ([[0]], 4000)
    pod7 = ([(40, 15, 0)], [[0]])
    case = (mt, rows, frac, option, {7: pod7}, [])
    assert check(DH, G, planes, case, 0)[0] == (po.EGS_ERR_TRANSACT, 4000, 0)
    case = (mt, rows, frac, option, {7: pod7}, [pod7 + (7,)])
    assert check(DH, G, planes, case, 0)[0] == (po.EGS_OK, 4000, 1)
    # the cached option is used even though the freed row would Trade elsewhere
    case = (mt, [(100, 40), (60, 25)], frac, ([[1]], 1), {}, [])
    assert check(DH, G, planes, case, 0)[0] == (po.EGS_OK, 1, 1 << 1)
    # "known not to fit": no victim applies (unknown uid, another node's pod) -> NOFIT; a whole-GPU victim frees it
    rows = [(0, 0), (20, 5)]
    whole = ([(0, 0, 1)], [[0]])
    assert check(DH, G, planes, (mt, rows, frac, None, {3: whole}, [whole + (4,)]), 0)[0] == (po.EGS_ERR_NOFIT, 0, 0)
    st_, _, masks = check(DH, G, planes, (mt, rows, frac, None, {3: whole}, [whole + (3,)]), 0)[0]
    assert st_ == po.EGS_OK and masks == 1
    # a repeated victim is forgotten once: two cancels of 40 cores would free a 70-core pod, one does not
    rows = [(10, 40)]
    pod5 = ([(40, 0, 0)], [[0]])
    assert check(DH, G, planes, (mt, rows, [(70, 1, 0)], None, {5: pod5}, [pod5 + (5,)] * 2), 1)[0][0] == po.EGS_ERR_NOFIT
    # a sentinel victim takes one core and one MiB back off its GPU
    rows = [(50, 20)]
    sent = ([SENT], [[0]])
    assert check(DH, G, planes, (mt, rows, frac, None, {9: sent}, [sent + (9,)]), 1)[0][0] == po.EGS_ERR_NOFIT
    assert check(DH, G, planes, (mt, rows, frac, None, {9: sent}, []), 1)[0][0] == po.EGS_OK
