"""A persistent in-process shard group (egs_comm_init_local) driven the way a host drives one, and the per-shard
checks the GPU tests make on it.

ShardGroup keeps one handle per rank and one long-lived worker thread per rank: every call on a rank is made from
that rank's own thread, across as many batches and verbs as a test likes.  `seq` runs a list of calls back to back on
every rank with no join across ranks in between; `each` is `seq` of one call.  Every check is per shard, on the owner
of the nodes it reads: after a sharded batch a rank's rows and option tables are current for its own range only.

Importing this module loads neither libegs nor a GPU."""
import queue
import threading

import numpy as np

from oracle_harness import compare_caches, compare_outputs, compare_rows, egs

JOIN_S = 600                                  # one call list on every rank; longer is a hang, not a slow batch


class ShardGroup:
    def __init__(self, cluster, world):
        cap = egs().capi
        self.world, self.n_nodes = world, cluster.n_nodes
        self.ranges = [cap.shard_range(cluster.n_nodes, r, world) for r in range(world)]
        self._jobs = [queue.Queue() for _ in range(world)]
        self._threads = [threading.Thread(target=self._work, args=(r,), daemon=True) for r in range(world)]
        self.hs = [None] * world
        for t in self._threads:
            t.start()

        def make(r, _):
            self.hs[r] = cluster.handle(world, r)
        self._run(range(world), [make])
        cap.comm_init_local(self.hs)

    # ---- driving
    def _work(self, r):
        while True:
            job = self._jobs[r].get()
            if job is None:
                return
            fns, out, done = job
            try:
                for fn in fns:
                    out.append(fn(r, self.hs[r]))
            except BaseException as ex:          # collected and raised on the caller's thread
                out.append(ex)
            done.set()

    def _run(self, ranks, fns):
        jobs = {}
        for r in ranks:
            jobs[r] = ([], threading.Event())
            self._jobs[r].put((list(fns), jobs[r][0], jobs[r][1]))
        errs = []
        for r, (out, done) in jobs.items():
            if not done.wait(JOIN_S):
                errs.append(f"rank {r}: no answer after {JOIN_S} s")
            elif out and isinstance(out[-1], BaseException):
                errs.append(f"rank {r}: {out[-1]!r}")
        assert not errs, "; ".join(errs)
        return [jobs[r][0] for r in ranks]

    def seq(self, fns):
        """fns[k](rank, handle) on every rank, back to back on each rank's thread; returns [rank][k] results."""
        return self._run(range(self.world), fns)

    def each(self, fn):
        """fn(rank, handle) on every rank; returns the results by rank."""
        return [res[0] for res in self.seq([fn])]

    def on(self, r, fn):
        """fn(rank, handle) on rank r alone (a call addressed to one rank, e.g. the owner of a node)."""
        return self._run([r], [fn])[0][0]

    def on_owner(self, node, fn):
        return self.on(self.owner(node), fn)

    # ---- layout
    def own(self, r):
        lo, hi = self.ranges[r]
        return range(lo, hi)

    def owner(self, node):
        for r, (lo, hi) in enumerate(self.ranges):
            if lo <= node < hi:
                return r
        raise ValueError(f"node {node} outside [0, {self.n_nodes})")

    def close(self):
        try:
            self.each(lambda r, h: h.close())
        finally:
            for q in self._jobs:
                q.put(None)
            for t in self._threads:
                t.join(timeout=60)
            assert not any(t.is_alive() for t in self._threads), "a rank's worker thread did not end"

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


# ------------------------------------------------------------------------------------------------ checks
def check_outputs(outs, ref, what, twin=None):
    """Every rank's outputs equal the oracle's (ref) and, when given, the unsharded twin's."""
    for r, out in enumerate(outs):
        compare_outputs(ref, out, f"{what}, rank {r} vs oracle")
        if twin is not None:
            compare_outputs(twin, out, f"{what}, rank {r} vs unsharded twin")


def sample_nodes(n_nodes, k, seed, extra=()):
    """Every node when there are at most k, else k sampled ones plus `extra` (e.g. the nodes a batch bound)."""
    if n_nodes <= k:
        return np.arange(n_nodes)
    rng = np.random.default_rng(seed)
    nodes = set(int(x) for x in rng.choice(n_nodes, k, replace=False)) | set(int(x) for x in extra if 0 <= x < n_nodes)
    return np.array(sorted(nodes), np.int64)


def check_shards(g, o, shapes=(), nodes=None, unfit_check=True):
    """Per shard, on its owner: the rows of the rank's own nodes, and the option cache of every shape in `shapes`,
    against the oracle.  `nodes` restricts both to a sample.  Ranks are checked one after the other, each on its
    own thread (the oracle is not shared across threads)."""
    keep = None if nodes is None else set(int(x) for x in nodes)
    for r in range(g.world):
        own = [n for n in g.own(r) if keep is None or n in keep]
        if not own:
            continue

        def check(_, h, own=own):
            compare_rows(h, o, own)
            if shapes:
                compare_caches(h, o, shapes, own, unfit_check=unfit_check)
        g.on(r, check)


def check_uids(g, o, uids, owner_of=None):
    """pod_known / pod_released of `uids` equal the oracle's on every rank; uids in owner_of (uid -> node, binds
    addressed to one rank) are checked on that node's owner only."""
    owner_of = owner_of or {}
    want = {int(u): (o.known_pod(int(u)), o.released_pod(int(u))) for u in list(uids) + list(owner_of)}
    common = [int(u) for u in uids if int(u) not in owner_of]

    def got(_, h, us):
        return {u: (h.pod_known(u), h.pod_released(u)) for u in us}
    for r, seen in enumerate(g.each(lambda r, h: got(r, h, common))):
        bad = [u for u in common if seen[u] != want[u]]
        assert not bad, f"rank {r}: pod_known / pod_released of uids {bad[:5]} differ from the oracle"
    for u, node in owner_of.items():
        seen = g.on_owner(node, lambda r, h: got(r, h, [u]))
        assert seen[u] == want[u], f"owner of node {node}: uid {u} known / released {seen[u]}, oracle {want[u]}"


# ------------------------------------------------------------------------------------------------ clusters, shapes
MEMS = (16384, 24576, 40960, 81920)          # MiB per GPU
FRAC_CORES = (0, 5, 10, 20, 25, 40, 50)


def hetero_nodes(rng, n_nodes):
    """Nodes of 1, 2, 4 or 8 GPUs of up to 81920 MiB; about half start partly used."""
    nodes = []
    for _ in range(n_nodes):
        g, m = int(rng.choice([1, 2, 4, 8])), int(rng.choice(MEMS))
        rows = None
        if rng.integers(0, 2):
            rows = ([int(rng.choice([100, 100, 60, 30, 0])) for _ in range(g)], [int(rng.integers(0, m + 1)) for _ in range(g)])
        nodes.append((g, m, rows))
    return nodes


def _frac(rng):
    return (int(rng.choice(FRAC_CORES)), 256 * int(rng.integers(1, 161)), 0)


def _unit(rng):
    k = rng.integers(0, 8)
    if k == 0:
        return (-1, -1, 0)
    if k == 1:
        return (0, 0, int(rng.integers(1, 3)))
    return _frac(rng)


def mixed_shapes(rng, n, single_share=0.5, avoid=()):
    """n distinct shapes, new against `avoid`: about single_share of them one fractional container (the resolver's
    fast path), the rest 1-4 containers mixing fractional, whole-GPU and no-GPU ({-1, -1}) units."""
    out, seen = [], set(avoid)
    while len(out) < n:
        if rng.random() < single_share:
            sh = (_frac(rng),)
        else:
            sh = tuple(_unit(rng) for _ in range(int(rng.integers(1, 5))))
        if sh not in seen:
            seen.add(sh); out.append(sh)
    return out


# ------------------------------------------------------------------------------------------------ the GPU cases
# Round-set batches at the new world sizes, each named by the resolver geometry it is chosen to reach (mw_geometry,
# csrc/egs_rounds.cuh; tests/test_shard_groups_host.py proves each claim on the CPU):
#   "trunc"  one round set whose shard lists the resolver truncates in shared memory (rke < rkm, `more` set)
#   "i96"    one round set of 96 shapes (MwInst96, the shallowest lists)
#   "host"   more than 96 shapes: the host forms the set of every round
ROUND_SET_CASES = [
    (3, 48, "trunc"), (3, 96, "i96"), (3, 200, "host"),
    (5, 32, "trunc"), (5, 96, "i96"), (5, 200, "host"),
    (6, 31, "trunc"), (6, 96, "i96"), (6, 200, "host"),
    (7, 32, "trunc"), (7, 96, "i96"), (7, 200, "host"),
]

# Shard layouts: (nodes, world, what the layout is chosen for)
LAYOUT_CASES = [
    (300, 7, "empty shards"),                 # ranks 0, 1, 3, 4 own nothing, the last shard 44 nodes
    (1, 8, "one node"),                       # every rank but the last owns nothing
    (128 * 3, 3, "128 w"), (128 * 3 + 1, 3, "128 w + 1"),
    (128 * 5, 5, "128 w"), (128 * 5 + 1, 5, "128 w + 1"),
    (128 * 8, 8, "128 w"), (128 * 8 + 1, 8, "128 w + 1"),
]

# State across batches on a group: (shapes already interned, new shapes) per batch.  The shape counts 12, 28, 60,
# 140, 16, 96 cross the 16 / 32 / 96 / host-formed geometries, so candidate buffers and CTA lists are reallocated.
STATE_WORLDS = (3, 5, 8)
STATE_PLAN = [(0, 12), (8, 20), (20, 40), (40, 100), (10, 6), (60, 36)]


def round_set_ns(n_shapes):
    """Shapes of the round set the resolver is configured for: the batch's, or RSMAX for host-formed sets."""
    return min(n_shapes, 96)
