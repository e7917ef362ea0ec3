"""On the CPU: the GPU cases of tests/test_gpu_shard_groups.py reach what their names claim, and the per-shard checks
of tests/shard_groups.py can fail.

- The resolver geometry (mw_geometry in csrc/egs_rounds.cuh, the function batch_rounds calls) compiled for the host:
  every round-set case hits its geometry class at its world size.
- The shard layouts give the stated empty and short shards.
- check_shards on oracle-made dumps: a one-cell change on a rank's own range fails, the same change outside it
  passes (a rank's state outside its range is not current after a sharded batch)."""
import copy
import ctypes as C

import numpy as np
import pytest

from oracle_harness import Cluster, egs
from shard_groups import LAYOUT_CASES, ROUND_SET_CASES, STATE_PLAN, check_shards, hetero_nodes, mixed_shapes, \
    round_set_ns

RKM = {16: 128, 32: 64, 96: 32}              # list depth of each resolver instance, by its shape capacity


@pytest.fixture(scope="module")
def geometry():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_rgeom())
    L.egsrg_geometry.argtypes = [C.c_int, C.c_int, C.c_void_p]

    def geo(ns, D):
        out = (C.c_longlong * 5)()
        assert L.egsrg_geometry(ns, D, out) == 0
        return dict(zip(["rkm", "rke", "pre_h", "pre_cap", "smem"], (int(x) for x in out)))
    geo.smem_max = L.egsrg_smem_max()
    return geo


def test_geometry_table(geometry):
    """The list depths of the world sizes the GPU cases run, and the limits every geometry respects."""
    want_rke = {  # D: rke at 16, 31, 32, 33, 48, 96 shapes
        3: [64, 64, 64, 32, 30, 14], 5: [64, 62, 60, 26, 18, 8], 6: [64, 52, 50, 22, 14, 6],
        7: [64, 44, 42, 18, 12, 6], 8: [60, 38, 36, 16, 10, 4]}
    for D, rkes in want_rke.items():
        assert [geometry(ns, D)["rke"] for ns in (16, 31, 32, 33, 48, 96)] == rkes, D
    assert geometry(16, 7)["smem"] == 227760
    assert geometry(16, 8)["pre_h"] == 30 and geometry(16, 3)["pre_h"] == 32
    for D in range(1, 9):
        for ns in range(1, 97):
            g = geometry(ns, D)
            inst = 16 if ns <= 16 else 32 if ns <= 32 else 96
            assert g["rkm"] == (min(RKM[inst], 64) if D > 2 else RKM[inst])
            assert 4 <= g["rke"] <= g["rkm"] and g["rke"] % 2 == 0
            assert g["smem"] <= geometry.smem_max
            if inst == 96:                           # no pre-install in the 96-shape resolver
                assert g["pre_h"] == 0 and g["pre_cap"] == 0
            else:
                nt = 512 if inst == 16 else 256
                assert g["pre_h"] == max(1, min(nt // ns, g["rke"] // 2)) and g["pre_cap"] == 3 * nt // 4


@pytest.mark.parametrize("world,n_shapes,kind", ROUND_SET_CASES)
def test_round_set_cases_reach_their_geometry(geometry, world, n_shapes, kind):
    g = geometry(round_set_ns(n_shapes), world)
    if kind == "trunc":
        assert g["rke"] < g["rkm"], g
        assert n_shapes <= 96
    elif kind == "i96":
        assert n_shapes == 96 and g["rkm"] == 32, g
    else:
        assert kind == "host" and n_shapes > 96
    # every new world size truncates somewhere among its cases, which the old world sizes 2 and 4 never do at 32
    assert any(geometry(round_set_ns(n), world)["rke"] < geometry(round_set_ns(n), world)["rkm"]
               for w, n, _ in ROUND_SET_CASES if w == world)


def test_state_plan_crosses_every_geometry():
    """The batches of the state-across-batches test: 1-16, 17-32, 33-96 and host-formed shape counts."""
    counts, interned = [], 0
    for n_old, n_new in STATE_PLAN:
        counts.append(min(n_old, interned) + n_new)
        interned += n_new
    classes = {0 if c <= 16 else 1 if c <= 32 else 2 if c <= 96 else 3 for c in counts}
    assert classes == {0, 1, 2, 3}, counts


def test_layouts(egs):
    cap = egs
    ranges = {(n, w): [cap.shard_range(n, r, w) for r in range(w)] for n, w, _ in LAYOUT_CASES}
    sizes = {k: [hi - lo for lo, hi in v] for k, v in ranges.items()}
    assert sizes[(300, 7)] == [0, 0, 128, 0, 0, 128, 44]
    assert sizes[(1, 8)] == [0] * 7 + [1]
    for w in (3, 5, 8):
        assert sizes[(128 * w, w)] == [128] * w
        assert sizes[(128 * w + 1, w)] == [128] * (w - 1) + [129]


# ------------------------------------------------------------------------------------------------ check self-test
class _Dump:
    """What a library handle would dump for the oracle `o`: state_dump and option_dump of every node."""

    def __init__(self, o, shapes):
        cap = egs().capi
        self.g_max, n = 8, o.n_nodes
        self.core = np.full((n, cap.row_width(8)), cap.EGS_PAD, np.int32)
        self.mem, self.gc = self.core.copy(), np.zeros(n, np.int32)
        for i in range(n):
            rows = o.rows(i)
            self.gc[i] = len(rows)
            self.core[i, :len(rows)], self.mem[i, :len(rows)] = zip(*rows)
        self.opts = {}
        for sh in shapes:
            present, score, masks = o.peek_many(range(n), sh)
            st = np.where(present, 1, np.where(o.trade_fits(range(n), sh), 0, 2)).astype(np.uint8)
            self.opts[tuple(sh)] = (st, score.astype(np.int32), masks.astype(np.uint8))

    def state_dump(self):
        return self.core, self.mem, self.gc, np.zeros_like(self.gc)

    def option_dump(self, req):
        return self.opts[tuple(req)]


class _Group:
    """ShardGroup's layout and `on` over dumps instead of handles."""

    def __init__(self, dumps, ranges):
        self.hs, self.ranges, self.world = dumps, ranges, len(dumps)

    def own(self, r):
        return range(*self.ranges[r])

    def on(self, r, fn):
        return fn(r, self.hs[r])


def _edits():
    """One-cell changes of a dump at node n: a row cell, a cached score, a cached mask, a presence."""
    def core(d, n, sh): d.core[n, 0] += 1
    def mem(d, n, sh): d.mem[n, d.gc[n] - 1] -= 1
    def score(d, n, sh): d.opts[sh][1][n] += 1
    def mask(d, n, sh): d.opts[sh][2][n, 0] ^= 1
    def state(d, n, sh): d.opts[sh][0][n] = 0 if d.opts[sh][0][n] == 1 else 1
    return [core, mem, score, mask, state]


def test_check_shards_fails_inside_own_range_only(egs):
    cap = egs
    rng = np.random.default_rng(5)
    n_nodes, world = 512, 3                                  # shards of 128, 128 and 256 nodes
    cl = Cluster(0, hetero_nodes(rng, n_nodes))
    shapes = mixed_shapes(rng, 3, single_share=1.0)
    o, o_lib = cl.oracle(), cl.oracle()
    for sh in shapes:                                       # cached options everywhere a shape fits
        for x in (o, o_lib):
            x.filter(None, list(sh))
    ranges = [cap.shard_range(n_nodes, r, world) for r in range(world)]
    base = _Dump(o_lib, shapes)
    check_shards(_Group([base] * world, ranges), o, shapes)
    for edit in _edits():
        for r in range(world):
            lo, hi = ranges[r]
            sh = shapes[0]
            cached = np.flatnonzero(base.opts[sh][0] == 1)
            inside = int(cached[(cached >= lo) & (cached < hi)][0])
            outside = int(cached[(cached < lo) | (cached >= hi)][0])
            for node, must_fail in ((inside, True), (outside, False)):
                d = copy.deepcopy(base)
                edit(d, node, sh)
                dumps = [base] * world
                dumps[r] = d
                if must_fail:
                    with pytest.raises(AssertionError):
                        check_shards(_Group(dumps, ranges), o, shapes)
                else:
                    check_shards(_Group(dumps, ranges), o, shapes)


def test_oracle_node_reset():
    """The oracle's node reload, which the GPU tests mirror egs_node_set_allocatable / egs_state_load_bulk with: new
    size and rows, the node's cached options gone, other nodes and podMaps untouched."""
    import oracle_c as oc
    o = oc.OracleC(0)
    for _ in range(2):
        o.add_node(400, 4 * 8192)
    sh = [(20, 1024, 0)]
    assert o.filter(None, sh).all()
    st, alloc = o.bind(0, sh, 5)
    assert st == 0 and o.known_pod(5)
    assert o.node_reset(0, 200, 2 * 4096, [50, 100], [1000, 4096]) == 0
    assert o.rows(0) == [(50, 1000), (100, 4096)]
    assert o.peek(0, sh) is None and o.peek(1, sh) is not None
    assert o.known_pod(5)
    assert o.add_pod(0, sh, [[1]], 6) == 0 and o.rows(0) == [(50, 1000), (80, 3072)]
    assert o.node_reset(0, 50, 100) == -1 and o.rows(0) == [(50, 1000), (80, 3072)]
