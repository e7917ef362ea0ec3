"""The comparisons of tests/oracle_harness.py, on the CPU.  Both sides come from the C oracle, the library side in the
shape of libegs's dumps (rows padded with EGS_PAD, option_dump at the handle's mask width, the six per-pod outputs).
Every comparison passes on equal input and raises on each single-cell change."""
import numpy as np
import pytest

from oracle_harness import FIELDS, Cluster, compare_caches, compare_outputs, compare_rows, compare_shards, egs, \
    oracle_batch

PODS = [((30, 4, 0),), ((0, 0, 1),), ((10, 2, 0), (-1, -1, 0))]
SHAPES = [((10, 2, 0),), ((20, 1, 0), (0, 0, 1), (5, 1, 0))]       # cached on the even nodes only


class Dump:
    """What a library handle of width g_max would dump for the oracle `o`: state_dump and option_dump."""

    def __init__(self, o, g_max):
        cap = egs().capi
        self.g_max, self.n_masks, n = g_max, 4, o.n_nodes
        self.core = np.full((n, cap.row_width(g_max)), cap.EGS_PAD, np.int32)
        self.mem, self.gc = self.core.copy(), np.zeros(n, np.int32)
        for i in range(n):
            rows = o.rows(i)
            self.gc[i] = len(rows)
            self.core[i, :len(rows)], self.mem[i, :len(rows)] = zip(*rows)
        self.opts = {}
        for sh in SHAPES:
            present, score, masks = o.peek_many(range(n), sh)
            st = np.where(present, 1, np.where(o.trade_fits(range(n), sh), 0, 2)).astype(np.uint8)
            self.opts[sh] = (st, score.astype(np.int32), masks.astype(cap.mask_dtype(g_max)))

    def state_dump(self):
        return self.core, self.mem, self.gc, np.zeros_like(self.gc)

    def option_dump(self, req):
        return self.opts[tuple(req)]


def _sides(g_max):
    """(oracle, library-side dump, the oracle's outputs, the library's outputs) after the same pods on both."""
    rng = np.random.default_rng(g_max)
    nodes = []
    for _ in range(24):
        g = int(rng.choice([1, 2, 4, 8] if g_max == 8 else [1, 2, 9, 12, 16]))
        core = [int(rng.choice([100, 100, 60, 30])) for _ in range(g)]
        rows = (core, [16 if c == 100 else int(rng.integers(4, 17)) for c in core])
        nodes.append((g, 16, rows if rng.integers(0, 2) else None))
    pick = rng.integers(0, len(PODS), 40)
    units = np.array([u for p in pick for u in PODS[p]], np.int32)
    c_off = np.concatenate([[0], np.cumsum([len(PODS[p]) for p in pick])]).astype(np.int32)
    uids = np.arange(1, len(pick) + 1, dtype=np.uint64)
    cl = Cluster(0, nodes, g_max)
    outs, dumps = [], []
    for o in (cl.oracle(), cl.oracle()):
        outs.append(oracle_batch(o, c_off, units, uids))
        for sh in SHAPES:
            o.filter(np.arange(0, len(nodes), 2), sh)
        dumps.append(o)
    o, lib = dumps[0], Dump(dumps[1], g_max)
    return o, lib, outs[0], outs[1]


def _check_all(o, lib, ref, got):
    n = len(lib.gc)
    compare_rows(lib, o, range(n))
    compare_caches(lib, o, SHAPES, range(n), unfit_check=True)
    compare_outputs(ref, got, "outputs")
    half = n // 2
    ranks = [(dict(got), lo, lib.core[lo:hi].copy(), lib.mem[lo:hi].copy()) for lo, hi in ((0, half), (half, n))]
    compare_shards(ref, (lib.core, lib.mem), ranks, "shards")
    return ranks


def _node(lib, want):
    """The first node of the multi-container shape's dump whose option state is `want`."""
    st = lib.opts[SHAPES[1]][0]
    i = np.flatnonzero(st == want)
    assert i.size, f"no node in state {want}"
    return int(i[0])


CHANGES = ["row", "pad", "presence", "score", "mask", "planes", "unfit", "rank_output", "shard_row"] + [f"output_{f}" for f in FIELDS]


@pytest.mark.parametrize("g_max", [8, 16])
def test_equal_sides_pass(g_max):
    o, lib, ref, got = _sides(g_max)
    _check_all(o, lib, ref, got)
    st = lib.opts[SHAPES[1]][0]
    assert (st == 0).any() and (st == 1).any() and (st == 2).any()    # all three states are compared


@pytest.mark.parametrize("change", CHANGES)
@pytest.mark.parametrize("g_max", [8, 16])
def test_single_cell_change_fails(g_max, change):
    o, lib, ref, got = _sides(g_max)
    n = len(lib.gc)
    st, sc, am = lib.opts[SHAPES[1]]
    short = int(np.flatnonzero(lib.gc < lib.core.shape[1])[0])
    if change == "row":
        lib.core[3, 0] += 1
    elif change == "pad":
        lib.mem[short, lib.gc[short]] = 0
    elif change == "presence":
        st[_node(lib, 1)] = 0
    elif change == "score":
        sc[_node(lib, 1)] += 1
    elif change == "mask":
        am[_node(lib, 1), 2] ^= 1 << (8 * am.itemsize - 1)          # the top GPU of container 2
    elif change == "planes":
        lib.n_masks = 8                                               # 4 planes dumped by an 8-plane handle
    elif change == "unfit":
        st[_node(lib, 0)] = 2                                         # a node that fits, marked "does not fit"
    elif change.startswith("output_"):
        got[change[len("output_"):]][17] += 1
    if change in ("rank_output", "shard_row"):
        ranks = _check_all(o, lib, ref, got)
        if change == "rank_output":
            ranks[1][0]["fit_count"] = ranks[1][0]["fit_count"].copy()
            ranks[1][0]["fit_count"][5] += 1
        else:
            ranks[1][2][n // 2 - 1, 0] += 1
        with pytest.raises(AssertionError):
            compare_shards(ref, (lib.core, lib.mem), ranks, "shards")
        return
    with pytest.raises(AssertionError):
        _check_all(o, lib, ref, got)
