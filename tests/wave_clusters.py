"""Planted clusters larger than one k_select wave, for the GPU tests of tests/test_gpu_large_clusters.py and their CPU
self-test tests/test_wave_clusters_host.py.  A helper module, not a test module.

k_select (egs_rounds.cuh) gives every warp 128-node chunks with a stride of the grid's warp count, and select_grid
(egs_rounds_impl.cuh) caps the grid at two CTAs of SEL_WARPS warps per SM.  So a warp handles a second chunk only when
a shard holds more than wave(n_sm) = 1024 * n_sm nodes; below that each warp's top-32 list and aggregates are built
from a single chunk.  Every case below is built to fail when the state a warp carries from one chunk to the next is
lost, and names that defect as a `mutant`: a transformation of the cluster under which the correct engine answers
as the defective engine answers on the planted cluster.

Every generator is seeded and prefix-stable: node i's rows depend on (seed, i, n_sm) only, never on the cluster
size, and a batch of fewer pods is a prefix of a longer one.  Arrays are built with numpy, never node by node."""
from dataclasses import dataclass
from typing import Callable

import numpy as np

from oracle_harness import Cluster

# egs_rounds.cuh / egs_rounds_impl.cuh geometry of k_select: SEL_THREADS / 32 warps per CTA, 128 nodes per chunk,
# at most 2 CTAs per SM
SEL_WARPS = 4
CHUNK = 128
CTAS_PER_SM = 2

G, M = 8, 64                        # every planted node: 8 GPUs of 100 core and M memory units each


def select_ctas(n_nodes, n_sm):
    """select_grid of egs_rounds_impl.cuh for a shard of n_nodes nodes."""
    chunks = (n_nodes + CHUNK - 1) // CHUNK
    return max(1, min((chunks + SEL_WARPS - 1) // SEL_WARPS, CTAS_PER_SM * n_sm))


def wave(n_sm):
    """Nodes k_select covers with one chunk per warp at the full grid (CTAS_PER_SM * SEL_WARPS * CHUNK per SM)."""
    return CTAS_PER_SM * SEL_WARPS * CHUNK * n_sm


def chunks_per_warp(n_nodes, n_sm):
    """The largest number of chunks any warp of k_select handles on a shard of n_nodes nodes (warp 0's count)."""
    chunks = (n_nodes + CHUNK - 1) // CHUNK
    return -(-chunks // (SEL_WARPS * select_ctas(n_nodes, n_sm)))


def chunk_geometry(n_nodes, n_sm):
    """Per node: its warp and its pass (which of that warp's chunks it lies in), and per node whether its chunk is
    the last one its warp handles."""
    nwarps = SEL_WARPS * select_ctas(n_nodes, n_sm)
    chunk = np.arange(n_nodes) // CHUNK
    n_chunks = (n_nodes + CHUNK - 1) // CHUNK
    last = chunk + nwarps >= n_chunks
    return chunk % nwarps, chunk // nwarps, last


@dataclass
class Rows:
    """A cluster of identical 8-GPU nodes with its rows: what Cluster.of_workload loads in bulk."""
    policy: int
    core: np.ndarray                # int32 [n_nodes, G]
    mem: np.ndarray                 # int32 [n_nodes, G]
    gpus: int = G
    mem_total: int = M

    @property
    def n_nodes(self):
        return self.core.shape[0]


def rows_cluster(policy, core, mem, g_max=8):
    return Cluster.of_workload(Rows(policy, np.ascontiguousarray(core, np.int32), np.ascontiguousarray(mem, np.int32)),
                               g_max)


@dataclass
class Planted:
    name: str
    cluster: Cluster
    c_off: np.ndarray               # int32 [P + 1]
    units: np.ndarray               # int32 [sum C, 3]
    mutant: Callable                # Cluster -> Cluster: the defect, as a transformation of the cluster
    mutant_doc: str
    shapes: list                    # the batch's distinct shapes

    @property
    def n_nodes(self):
        return self.cluster.n_nodes


# ------------------------------------------------------------------------------------------------ helpers
def _hash(seed, salt, idx):
    """splitmix64 of (seed, salt, node index), vectorised: a prefix-stable per-node random stream."""
    with np.errstate(over="ignore"):
        z = np.asarray(idx, np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64((seed * 1000003 + salt) & (2**64 - 1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def _pick(seed, salt, n_nodes, choices, per_gpu=True):
    """Per node (and per GPU when per_gpu) a value from `choices`, prefix-stable."""
    idx = np.arange(n_nodes, dtype=np.uint64)
    if per_gpu:
        idx = (idx[:, None] * np.uint64(G) + np.arange(G, dtype=np.uint64)[None, :])
    return np.asarray(choices, np.int32)[(_hash(seed, salt, idx) % np.uint64(len(choices))).astype(np.int64)]


def _batch(shapes, picks):
    units = [u for p in picks for u in shapes[int(p)]]
    c_off = np.concatenate([[0], np.cumsum([len(shapes[int(p)]) for p in picks])]).astype(np.int32)
    return c_off, np.array(units, np.int32).reshape(-1, 3)


def _picks(seed, n_shapes, n_pods, lead=()):
    """`lead` first, then every shape once in a seeded order, then seeded picks (prefix-stable in n_pods)."""
    rng = np.random.default_rng(seed)
    order = list(lead) + [int(s) for s in rng.permutation(n_shapes)]
    order += [int(s) for s in rng.integers(0, n_shapes, max(0, n_pods - len(order)))]
    return order[:n_pods]


def truncate_at_wave(n_sm):
    """Mutant "the second pass is invisible": every node of a second or later chunk of its warp is dropped, as if it
    were unfit.  At the full grid those are exactly the nodes >= wave(n_sm)."""
    def mut(cl):
        w = cl.workload
        k = min(w.n_nodes, wave(n_sm))
        return rows_cluster(w.policy, w.core[:k], w.mem[:k], cl.g_max)
    return mut


DEAD = (0, 0)                       # every GPU at core 0 and mem 0: no shape of these batches fits


def only_last_chunk(n_sm):
    """Mutant "each warp's list is reset at every chunk": a node in a chunk before its warp's last one cannot win, as
    if it were unfit (the fit count and digests of the defect still count it; the winner is what tells them apart)."""
    def mut(cl):
        w = cl.workload
        _, _, last = chunk_geometry(w.n_nodes, n_sm)
        core, mem = w.core.copy(), w.mem.copy()
        core[~last], mem[~last] = DEAD
        return rows_cluster(w.policy, core, mem, cl.g_max)
    return mut


# ------------------------------------------------------------------------------------------------ the cases
A_SHAPES = [((20, 8, 0),), ((50, 16, 0),), ((0, 0, 1),), ((10, 4, 0), (0, 0, 1)), ((30, 8, 0), (-1, -1, 0))]


def case_a(n_nodes, n_sm, policy, n_pods=256, seed=1):
    """A, only beyond the wave: every node below wave(n_sm) has all GPUs at core 0, so no shape of the batch fits it.
    Node W = wave(n_sm) always fits; about a third of the nodes past it fit, with seeded rows."""
    W = wave(n_sm)
    full = np.arange(n_nodes) >= W
    fit = full & ((_hash(seed, 1, np.arange(n_nodes)) % np.uint64(3) == 0) | (np.arange(n_nodes) == W))
    core = np.where(fit[:, None], _pick(seed, 2, n_nodes, [100, 100, 100, 70, 40, 0]), 0)
    mem = np.where(fit[:, None], _pick(seed, 3, n_nodes, [M, M, M, 48, 20, 8]), _pick(seed, 4, n_nodes, [M, 30]))
    core[fit, 0], mem[fit, 0] = 100, M          # GPU 0 free: every fit node fits each single-container shape
    c_off, units = _batch(A_SHAPES, _picks(seed, len(A_SHAPES), n_pods))
    return Planted("A", rows_cluster(policy, core, mem), c_off, units, truncate_at_wave(n_sm),
                   "second pass invisible", A_SHAPES)


B_SHAPES = [((20, 4, 0),), ((10, 16, 0),), ((0, 0, 1),), ((5, 2, 0), (5, 2, 0))]


def case_b(n_nodes, n_sm, policy, n_pods=256, seed=2):
    """B, best beyond the wave: every node below wave(n_sm) is whole on core and at mem 8 on every GPU, so it fits
    the shapes asking for little memory with a low binpack score, and not (10, 16) or a whole GPU.  Every node past the
    wave has GPU 0 free and seeded use on the others: it fits every shape, with the highest binpack scores."""
    W = wave(n_sm)
    past = np.arange(n_nodes) >= W
    core = np.where(past[:, None], _pick(seed, 1, n_nodes, [100, 60, 30, 0]), 100)
    mem = np.where(past[:, None], _pick(seed, 2, n_nodes, [M, 40, 12, 0]), 8)
    core[past, 0], mem[past, 0] = 100, M
    c_off, units = _batch(B_SHAPES, _picks(seed, len(B_SHAPES), n_pods, lead=(0, 1, 2)))
    return Planted("B", rows_cluster(policy, core, mem), c_off, units, truncate_at_wave(n_sm),
                   "second pass invisible", B_SHAPES)


C_SHAPES = [((20, 4, 0),)]


def case_c(n_nodes, n_sm, policy, n_pods=400, seed=3):
    """C, ties across passes.  Top nodes (GPU 0 free, the others empty) share the top binpack key of (20, 4) and fall
    from it after one bind; plain nodes (all GPUs free) score lower; dead nodes do not fit.  The first chunk of every
    odd warp is dead, so that warp's lowest fit ids come from its second chunk; the first chunk of every even warp and
    every later chunk are plain with seeded top nodes, more than 128 of them in all.  Under spread every fit node ties
    and the winner is the lowest fit id."""
    warp, pas, _ = chunk_geometry(max(n_nodes, wave(n_sm) + 1), n_sm)
    warp, pas = warp[:n_nodes], pas[:n_nodes]
    k = min(CHUNK, max(2, -(-160 // (wave(n_sm) // CHUNK // 2))))       # top nodes per chunk
    top = _hash(seed, 1, np.arange(n_nodes)) % np.uint64(CHUNK) < np.uint64(k)
    top |= (pas >= 1) & (np.arange(n_nodes) % CHUNK == 0)              # node W among them
    dead = (pas == 0) & (warp % 2 == 1)
    top &= ~dead
    core = np.full((n_nodes, G), 100, np.int32)
    mem = np.full((n_nodes, G), M, np.int32)
    core[top, 1:], mem[top, 1:] = 0, 0
    core[dead], mem[dead] = DEAD
    c_off, units = _batch(C_SHAPES, [0] * n_pods)
    return Planted("C", rows_cluster(policy, core, mem), c_off, units, only_last_chunk(n_sm),
                   "list reset at every chunk", C_SHAPES)


def d_shapes(n_shapes, seed):
    """n_shapes distinct shapes, 1 or 2 containers: fractional, whole-GPU and {-1, -1} units."""
    rng = np.random.default_rng(seed)
    out, seen = [], set()
    while len(out) < n_shapes:
        sh = []
        for _ in range(1 if rng.random() < 0.75 else 2):
            k = rng.random()
            if k < 0.1:
                sh.append((-1, -1, 0))
            elif k < 0.3:
                sh.append((0, 0, int(rng.integers(1, 3))))
            else:
                sh.append((int(rng.choice([5, 10, 20, 30, 50])), int(rng.integers(1, 25)), 0))
        sh = tuple(sh)
        if sh not in seen:
            seen.add(sh); out.append(sh)
    return out


def case_d(n_nodes, n_sm, policy, n_shapes=40, n_pods=None, seed=4):
    """D, many shapes past the wave: n_shapes distinct shapes (40: groups of 32 inside each chunk; 110: more than a
    round set of 96, so host-formed round sets and the cold evaluate's break).  Nodes below the wave are nearly full
    with seeded use; nodes past it have more room, so the fit sets of most shapes cross the wave."""
    W = wave(n_sm)
    past = (np.arange(n_nodes) >= W)[:, None]
    core = np.where(past, _pick(seed, 1, n_nodes, [100, 100, 60, 30, 0]), _pick(seed, 2, n_nodes, [100, 30, 10, 0, 0, 0]))
    mem = np.where(past, _pick(seed, 3, n_nodes, [M, M, 40, 16, 4]), _pick(seed, 4, n_nodes, [M, 12, 6, 2, 0]))
    shapes = d_shapes(n_shapes, seed)
    c_off, units = _batch(shapes, _picks(seed, n_shapes, n_pods or n_shapes + 12))
    return Planted(f"D{n_shapes}", rows_cluster(policy, core, mem), c_off, units, truncate_at_wave(n_sm),
                   "second pass invisible", shapes)


CASES = {"A": case_a, "B": case_b, "C": case_c, "D40": lambda *a, **k: case_d(*a, n_shapes=40, **k),
         "D110": lambda *a, **k: case_d(*a, n_shapes=110, **k)}


def sizes(n_sm):
    """The two planted sizes: one node in warp 0's second chunk, and a partial third chunk."""
    W = wave(n_sm)
    return [W + 1, 2 * W + 127]
