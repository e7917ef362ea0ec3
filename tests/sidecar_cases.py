"""Planted clusters for the leaf-split Trade of a sidecar handle (egs_create_ex with c_max > 4), for the GPU tests of
tests/test_gpu_sidecar_scale.py and their CPU self-test tests/test_sidecar_cases_host.py.  A helper module, not a
test module.

A shape with more than 4 branching containers (fractional or sentinel units, one GPU digit each) on an 8-GPU sidecar
handle is Traded by k_trade_probe / k_trade_leaves / k_trade_commit (egs_kernels.cuh).  The leaf space of a node has
one 3-bit digit per branching container, the first container most significant (trade_leaf_eval); a tile is
LEAF_THREADS chunks of LEAF_CHUNK leaves, i.e. leaves [t * 2^14, (t + 1) * 2^14), and k_trade_leaves grid-strides
over the (miss, tile) items with at most 8 CTAs of LEAF_THREADS threads per SM.  Every planted node kind below names
the defect it catches as a `mutant`: a change of its rows under which the oracle's answer changes.

Every node has mem_total M per GPU; rows are seeded and built with numpy, never drawn from the device."""
from dataclasses import dataclass

import numpy as np

LEAF_THREADS, LEAF_CHUNK = 256, 64           # egs_kernels.cuh
TILE = LEAF_THREADS * LEAF_CHUNK             # leaves per (miss, tile) item
BITS = 3                                     # digit width on a handle with g_max 5..8
CTAS_PER_SM_MAX = 2048 // LEAF_THREADS       # 2048 resident threads per SM: no occupancy gives more
M = 32
SENT = (-1, -1, 0)

# Leaf-split shapes: 5, 6 and 8 branching containers (2, 16 and 1 024 tiles per miss).  Container 0 asks for 20 memory
# units, so the rows below steer the leading digit; (1, 8, 0) containers steer the next ones.
S5 = ((1, 20, 0), (0, 0, 1), (1, 8, 0), (1, 8, 0), SENT, SENT)
S6 = ((1, 20, 0), (1, 8, 0), (1, 8, 0), (1, 8, 0), SENT, SENT)
S8 = ((1, 20, 0), (1, 8, 0), (1, 8, 0), (1, 8, 0), SENT, SENT, SENT, SENT)
SPLIT = {5: S5, 6: S6, 8: S8}

# One-thread DFS shapes with 5..8 containers and at most 4 branching ones, and small shapes of 1..4 containers.
DFS = [
    ((10, 4, 0), (0, 0, 1), SENT, SENT, (0, 0, 1)),
    ((0, 0, 1), SENT, SENT, SENT, SENT),
    ((5, 2, 0), (0, 0, 2), SENT, (3, 1, 0), (0, 0, 1), SENT, (0, 0, 1)),
    ((20, 6, 0), SENT, (0, 0, 1), SENT, (10, 3, 0), (0, 0, 1), (0, 0, 1), (0, 0, 1)),
    (SENT, SENT, SENT, SENT, SENT),
]
SMALL = [((30, 8, 0),), ((0, 0, 1),), ((10, 4, 0), SENT), ((5, 2, 0), (0, 0, 1), SENT, SENT)]


def n_branch(shape):
    return sum(1 for u in shape if u[2] == 0)


def tiles(shape):
    """Tiles per miss of a shape on an 8-GPU sidecar handle (LeafArgs::tiles)."""
    return -(-(1 << (BITS * n_branch(shape))) // TILE)


def items(n_miss, shape):
    return n_miss * tiles(shape)


def leaf_grid_max(n_sm):
    """An upper bound of k_trade_leaves' grid (occupancy per SM times n_sm), whatever its register count."""
    return CTAS_PER_SM_MAX * n_sm


def several_items_per_cta(n_miss, shape, n_sm):
    """Every CTA of the grid takes at least three items, so items of different misses, at any occupancy."""
    return items(n_miss, shape) >= 3 * leaf_grid_max(n_sm)


def leaf_of(alloc, shape):
    """The leaf index of an allocation (one GPU list per container): digit j is the GPU of branching container j."""
    d = [a[0] for a, u in zip(alloc, shape) if u[2] == 0]
    leaf = 0
    for g in d:
        leaf = (leaf << BITS) | g
    return leaf


def tile_of(leaf):
    return leaf // TILE


def chunk_of(leaf):
    return leaf // LEAF_CHUNK


def warp_of(leaf):
    """tile * 8 + the warp of the CTA that evaluates the leaf."""
    return leaf // (32 * LEAF_CHUNK)


# ------------------------------------------------------------------------------------------------ node kinds
@dataclass
class Kind:
    name: str
    rows: list                  # [(core, mem)] per GPU, 5..8 GPUs
    mutant: list                # the rows under the defect's transformation
    doc: str


def _set(rows, g, v):
    r = list(rows)
    r[g] = v
    return r


_LATE = [(100, 4)] * 4 + [(100, 16)] * 3 + [(100, M)]
_TIE_TILE = [(100, M), (100, 8), (40, 8), (60, M), (40, 16), (60, 4), (60, M), (100, 24)]
_TIE_CHUNK = [(40, 0), (100, M), (20, 12), (20, 0), (20, 12), (60, 0), (60, 12), (0, M)]
_TIE_LANE = [(40, 12), (0, 0), (0, 24), (0, 16), (20, 8), (20, 8), (100, M), (100, 12)]
_EARLY = [(100, M), (100, M), (100, 0), (0, 8), (100, 16), (60, 8), (20, 8), (60, 16)]
_LATE_LOW = [(100, 0), (60, 0), (60, 0), (100, 0), (100, 8), (60, 8), (100, M), (100, M)]
_PREFIX = [(100, 4)] * 3 + [(100, 24)] * 2 + [(100, 12)] * 3
_ABSENT = [(100, M), (60, 12), (100, 24), (40, 8), (100, M), (20, 20), (100, 12)]

KINDS = {k.name: k for k in [
    Kind("late", _LATE, _set(_LATE, 7, (100, 16)),
         "S6: container 0 fits GPU 7 only and container 1 GPUs 4..7 only, so every feasible leaf lies in the last "
         "tile (S5's whole-GPU container finds no free GPU here; `late_low` is S5's late node).  Mutant: GPU 7 "
         "forbidden for container 0 (what a CTA that drops its later items sees)."),
    Kind("tie_tile", _TIE_TILE, _set(_TIE_TILE, 6, (60, 19)),
         "S6 binpack: GPUs 3 and 6 are twins; the best leaf puts container 0 alone on GPU 6, its twin on GPU 3 ties "
         "in another tile and the later one wins.  Mutant: GPU 6 too small for container 0, the winner moves."),
    Kind("tie_chunk", _TIE_CHUNK, _set(_TIE_CHUNK, 4, (20, 7)),
         "S6 binpack: twins 2 and 4 for branching container 2: the two maximal leaves lie in one tile, in chunks of "
         "different warps.  Mutant: GPU 4 too small for it."),
    Kind("tie_lane", _TIE_LANE, _set(_TIE_LANE, 5, (20, 7)),
         "S6 binpack: twins 4 and 5 for branching container 3: the two maximal leaves lie in two lanes of one warp.  "
         "Mutant: GPU 5 too small for it."),
    Kind("early", _EARLY, _EARLY,
         "Container 0 fits GPUs 0 and 1 only: an early best leaf with a high binpack score."),
    Kind("late_low", _LATE_LOW, _EARLY,
         "Container 0 fits GPUs 6 and 7 only: a late best leaf with a lower binpack score.  Alternating with "
         "`early`, a CTA that mixes two misses' keys changes a cached score or mask.  Mutant: all nodes equal."),
    Kind("unfit_first", [(100, 16)] * 8, _set([(100, 16)] * 8, 0, (100, M)),
         "No GPU takes container 0: no feasible leaf for S5 / S6 / S8.  Mutant: one free GPU more (S6 and S8 fit)."),
    Kind("unfit_whole", [(99, M)] * 8, _set([(99, M)] * 8, 0, (100, M)),
         "No free GPU for S5's whole-GPU container (S6 fits).  Mutant: one free GPU more."),
    Kind("prefix", _PREFIX, _set(_set(_PREFIX, 3, (100, 16)), 4, (100, 16)),
         "Container 0 fits GPUs 3 and 4 only and container 1 then GPUs 4..7: S6's first feasible leaf is 3 * 2^15 + "
         "4 * 2^12, after an infeasible run over six whole tiles and every chunk of the seventh.  Mutant: GPUs 3 "
         "and 4 too small for container 0 (nothing fits)."),
    Kind("absent5", _ABSENT[:5], _ABSENT[:5] + [(100, M)] * 3,
         "5 GPUs: digits 5..7 name absent GPUs, whose PAD rows fail every unit.  Mutant: the same node with 8 GPUs, "
         "the 3 more free."),
    Kind("absent6", _ABSENT[:6], _ABSENT[:6] + [(100, M)] * 2, "6 GPUs; mutant: 8 GPUs."),
    Kind("absent7", _ABSENT[:7], _ABSENT[:7] + [(100, M)], "7 GPUs; mutant: 8 GPUs."),
]}

# (kind, branching container, earlier twin, later twin) of the three tie kinds under binpack with S6
TIES = [("tie_tile", 0, 3, 6), ("tie_chunk", 2, 2, 4), ("tie_lane", 3, 4, 5)]
PLANTED = [k for k in KINDS if k not in ("early", "late_low")]


def node(rows):
    """A Cluster node entry: (gpu count, M, (core row, mem row))."""
    return (len(rows), M, ([c for c, _ in rows], [m for _, m in rows]))


def planted_cluster(n_nodes, mutate=None):
    """n_nodes nodes alternating `early` / `late_low`, with every planted kind at max(3, n_nodes // 96) positions spread
    evenly over the whole id range.  Returns (nodes, {kind: node ids}).  mutate: a kind whose nodes take their mutant
    rows (mutate="late_low": every bulk node is `early`)."""
    kind = np.where(np.arange(n_nodes) % 2 == 0, "early", "late_low").astype(object)
    per = max(3, n_nodes // 96)
    where = {}
    for q, k in enumerate(PLANTED):
        ids = np.arange(per) * n_nodes // per + 7 * q + 3
        kind[ids] = k
        where[k] = ids
    where["early"] = np.flatnonzero(kind == "early")
    where["late_low"] = np.flatnonzero(kind == "late_low")
    nodes = [node(KINDS[k].mutant if k == mutate else KINDS[k].rows) for k in kind]
    return nodes, where


def planted_nodes(n_sm):
    """A node count at which a cold Trade of S5 over every node gives each CTA of k_trade_leaves at least three items
    (S6 and S8 need fewer misses), with more than 256 misses and several probe blocks."""
    return max(300, -(-3 * leaf_grid_max(n_sm) // tiles(S5)) + 64)


def s8_count(n_sm):
    """Misses of S8 (1 024 tiles each) that give every CTA three items: at least 2."""
    return max(2, -(-3 * leaf_grid_max(n_sm) // tiles(S8)))


# ------------------------------------------------------------------------------------------------ batch clusters
def batch_cluster(n_nodes, seed):
    """Seeded nodes of 5..8 GPUs with varied use, on which most DFS and leaf-split shapes fit, and `champion` nodes --
    all GPUs free -- in the second and fourth 256-node blocks only: every champion ties on the best score of a DFS
    shape, so the first one must win over k_pass's block partials.  Returns (nodes, champion ids)."""
    rng = np.random.default_rng(seed)
    nodes = []
    for _ in range(n_nodes):
        g = int(rng.choice([8, 8, 8, 7, 6, 5]))
        core = rng.choice([100, 100, 60, 40, 20, 0], g).astype(int)
        mem = np.where(core == 100, M, rng.choice([24, 16, 12, 8, 4, 0], g)).astype(int)
        core[0], mem[0] = 100, M                          # container 0 of every leaf-split shape fits somewhere
        nodes.append((g, M, (core.tolist(), mem.tolist())))
    champ = [b * 256 + int(x) for b in (1, 3) for x in rng.integers(0, 256, 2) if b * 256 + int(x) < n_nodes]
    for i in champ:
        nodes[i] = (8, M, None)
    return nodes, sorted(set(champ))


def pods(rng, n_pods, split_every=4):
    """A batch: every split_every-th pod a leaf-split shape (S5 or S6), the others DFS and small shapes."""
    out = []
    for p in range(n_pods):
        if p % split_every == 0:
            out.append(list(S5 if rng.integers(0, 2) else S6))
        else:
            pool = DFS + SMALL
            out.append(list(pool[int(rng.integers(0, len(pool)))]))
    return out


def batch(pods_):
    c_off = np.cumsum([0] + [len(p) for p in pods_]).astype(np.int32)
    units = np.array([u for p in pods_ for u in p], np.int32).reshape(-1, 3)
    return c_off, units
