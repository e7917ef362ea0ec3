"""The sharded rounds engine on persistent in-process shard groups (tests/shard_groups.py), against the C oracle and
an unsharded twin handle driven by the same calls: the world sizes 3, 5, 6 and 7, empty and short shards, state
carried through many batches and the verbs between them, mutation streams, and batches issued back to back.

After a sharded round each rank writes back the tracked nodes of its own range (rows, option states, NEW -> CACHED /
ABSENT) and consumes the observation flags in its own k_merge.  A wrong state left there does not show in the batch
that wrote it, only in the next call that reads it; so every check here is per shard, on the owner, and most tests
run more than one batch on the same handles."""
import numpy as np
import pytest

import oracle_c as oc
from oracle_harness import FIELDS, Cluster, egs, oracle_mut
from round_batches import STOPS, Batch, distinct_shapes, pod_picks, stats_delta
from shard_groups import (LAYOUT_CASES, ROUND_SET_CASES, STATE_PLAN, STATE_WORLDS, ShardGroup, check_outputs,
                          check_shards, check_uids, hetero_nodes, mixed_shapes, sample_nodes)

pytestmark = pytest.mark.gpu
LIB = 0x8000000000000000                    # the first library-assigned uid


def _cap():
    return egs().capi


class LibUids:
    """The uids a handle assigns to the pods of batches without explicit uids: the same on every rank and on the
    twin (each starts at LIB and moves on by the batch's pods).  The oracle is given them explicitly, so that no
    batch reuses an earlier batch's uids there."""

    def __init__(self):
        self.next = LIB

    def take(self, n):
        u = np.arange(self.next, self.next + n, dtype=np.uint64)
        self.next += n
        return u


def _run_group_batch(g, twin, o, c_off, units, uids=None, lib=None, threads=4):
    """One batch on every rank of g, on the twin and on the oracle; checks the outputs and returns the oracle's.
    uids None: the library numbers the pods, and `lib` (a LibUids) says how."""
    o_uids = uids if uids is not None else lib.take(len(c_off) - 1)
    ref = o.schedule_batch(c_off, units.astype(np.int64), uids=o_uids, threads=threads)
    outs = g.each(lambda r, h: h.schedule_batch(c_off, units, uids=uids, mode=2))
    tw = twin.schedule_batch(c_off, units, uids=uids, mode=2) if twin is not None else None
    check_outputs(outs, ref, "batch", tw)
    return ref


# ------------------------------------------------------------------------------------------------ odd world sizes
CONFIG_CASES = [(4, 3000, 6000, None), (1, 2000, 4000, None), (2, 3000, 6000, None), (3, 300, 2000, 0), (4, 1000, 3000, 0)]


@pytest.mark.parametrize("world", [3, 5, 6, 7])
def test_config_cases_at_odd_world_sizes(world):
    """test_sharding's five config cases, reduced, at world sizes no other test runs: every rank's outputs equal the
    oracle's and the twin's, and every shard's rows and sampled option caches equal the oracle's."""
    eg = egs()
    for cfg, nn, npods, pol in CONFIG_CASES:
        w = eg.workloads.config(cfg, n_nodes=nn, n_pods=npods, policy=pol)
        cl = Cluster.of_workload(w)
        o, twin = cl.oracle(), cl.handle()
        with ShardGroup(cl, world) as g:
            ref = _run_group_batch(g, twin, o, w.c_off, w.units, lib=LibUids())
            nodes = sample_nodes(w.n_nodes, 600, cfg, ref["node"])
            check_shards(g, o, eg.workloads.shapes_of(w), nodes)
        twin.close()


@pytest.mark.parametrize("world,n_shapes,kind", ROUND_SET_CASES)
def test_round_sets_at_odd_world_sizes(world, n_shapes, kind):
    """Round sets chosen from the resolver geometry at this world size: truncated shard lists (rke < rkm), the
    96-shape set and host-formed sets.  Every one of them truncates the lists (rke < rkm): rounds must end on a
    dry list, and every rank's resolver must count the same rounds and stops."""
    rng = np.random.default_rng(world * 1000 + n_shapes)
    nodes = hetero_nodes(rng, 2500)
    shapes = mixed_shapes(rng, n_shapes)
    b = Batch(1, nodes, shapes, pod_picks(rng, shapes, 4000, "trickle" if kind == "host" else "front"))
    assert len(distinct_shapes(b)) == n_shapes
    o, twin = b.cluster.oracle(), b.cluster.handle()
    with ShardGroup(b.cluster, world) as g:
        s0 = g.each(lambda r, h: h.rounds_stats())
        ref = _run_group_batch(g, twin, o, b.c_off, b.units, lib=LibUids())
        d = [stats_delta(s1, s) for s1, s in zip(g.each(lambda r, h: h.rounds_stats()), s0)]
        assert all(x == d[0] for x in d), f"replicated resolvers differ in their stats: {d}"
        print(f"world {world}, {n_shapes} shapes ({kind}): {d[0]}")
        assert d[0]["pods"] == b.n_pods
        assert d[0]["stop_list_dry"] > 0, d[0]
        assert sum(d[0][k] for k in STOPS) == d[0]["rounds"], d[0]
        check_shards(g, o, distinct_shapes(b), sample_nodes(b.n_nodes, 500, n_shapes, ref["node"]))
    twin.close()


# ------------------------------------------------------------------------------------------------ shard layouts
@pytest.mark.parametrize("n_nodes,world,what", LAYOUT_CASES)
def test_shard_layouts(n_nodes, world, what):
    """Empty shards, a one-node cluster, and clusters of 128 w and 128 w + 1 nodes: two batches on the same group
    (the second reads the option tables the first wrote back), every node's rows and caches checked on its owner."""
    rng = np.random.default_rng(n_nodes * 10 + world)
    nodes = hetero_nodes(rng, n_nodes)
    shapes = mixed_shapes(rng, 20)
    cl = Cluster(0, nodes)
    o, twin = cl.oracle(), cl.handle()
    lib = LibUids()
    with ShardGroup(cl, world) as g:
        for k in range(2):
            b = Batch(0, nodes, shapes, pod_picks(rng, shapes, 3 * n_nodes + 40, "front"))
            _run_group_batch(g, twin, o, b.c_off, b.units, lib=lib)
            check_shards(g, o, shapes)
    twin.close()


# ------------------------------------------------------------------------------------------------ state across batches
class _Mirror:
    """The same calls on a shard group (every rank, or the owner), its unsharded twin and the oracle."""

    def __init__(self, g, twin, o, policy, nodes):
        self.g, self.twin, self.o, self.policy = g, twin, o, policy
        self.size = [(gc, mt) for gc, mt, _ in nodes]         # GPUs and memory per GPU of every node, as loaded

    def records(self, recs):
        assert all(st == 0 for st in self.g.each(lambda r, h: h.mutations_apply(recs)))
        assert self.twin.mutations_apply(recs) == 0
        for rec in recs:
            oracle_mut(self.o, rec)

    def filter_bind(self, ids, sh, uid, rng):
        """Filter on the owner of ids (all of one shard), then bind one fit node there."""
        fo = self.o.filter(ids, sh)
        fg = self.g.on_owner(int(ids[0]), lambda r, h: h.filter(ids, sh))
        assert np.array_equal(fg, fo) and np.array_equal(self.twin.filter(ids, sh), fo), f"filter {sh}"
        fit = ids[fo == 1]
        if not fit.size:
            return None
        node = int(fit[int(rng.integers(0, fit.size))])
        want = self.o.bind(node, sh, uid)
        assert self.g.on_owner(node, lambda r, h: h.bind(node, sh, uid)) == want, f"bind {sh} on node {node}"
        assert self.twin.bind(node, sh, uid) == want
        return node

    def node_set(self, node, gc, mt):
        assert all(st == 0 for st in self.g.each(lambda r, h: h.node_set_allocatable(node, 100 * gc, mt * gc)))
        assert self.twin.node_set_allocatable(node, 100 * gc, mt * gc) == 0
        assert self.o.node_reset(node, 100 * gc, mt * gc) == 0
        self.size[node] = (gc, mt)

    def load_bulk(self, node0, gc, mt, core, mem):
        self.g.each(lambda r, h: h.state_load_bulk(node0, gc, mt, core, mem))
        self.twin.state_load_bulk(node0, gc, mt, core, mem)
        for i in range(len(core)):
            assert self.o.node_reset(node0 + i, 100 * gc, mt * gc, core[i], mem[i]) == 0
            self.size[node0 + i] = (gc, mt)

    def restore(self):
        """A restarted scheduler on the current rows: empty option caches and pod maps on every side."""
        self.g.each(lambda r, h: (h.snapshot(), h.restore()))
        self.twin.snapshot(); self.twin.restore()
        fresh = oc.OracleC(self.policy)
        for n, (gc, mt) in enumerate(self.size):
            assert fresh.add_node(100 * gc, mt * gc) == n
            rows = self.o.rows(n)
            fresh.set_rows(n, [c for c, _ in rows], [m for _, m in rows])
        self.o = fresh


def _between(m, rng, interned, last, uid):
    """Every kind of call a host makes between two batches, on the right ranks.  Returns (next uid, owner-bound
    uids -> node)."""
    cap, g, o = _cap(), m.g, m.o
    # mutation records on every rank: AddPod, ForgetPod of pods the last batch placed, a failing AddPod then its
    # ForgetPod (the GPU ends above its totals), a sidecar
    recs = []
    for r in range(g.world):
        own = g.own(r)
        if not len(own):
            continue
        node = int(rng.integers(own.start, own.stop))
        gc = o.gpu_count(node)
        recs.append((cap.EGS_MUT_ADD, node, [(10, 512, 0)], [[int(rng.integers(0, gc))]], uid)); uid += 1
        full = [gi for gi, (c, _) in enumerate(o.rows(node)) if c < 100]
        gi = full[0] if full else 0
        recs.append((cap.EGS_MUT_ADD, node, [(0, 0, 1)], [[gi]], uid))              # whole GPU on a used one: fails
        recs.append((cap.EGS_MUT_FORGET, node, [(0, 0, 1)], [[gi]], uid)); uid += 1
        recs.append((cap.EGS_MUT_ADD, node, [(20, 1024, 0), (-1, -1, 0)], [[int(rng.integers(0, gc))], []], uid)); uid += 1
    placed = np.nonzero(last["status"] == 0)[0]
    for p in rng.choice(placed, min(6, placed.size), replace=False):
        sh = last["shapes"][p]
        recs.append((cap.EGS_MUT_FORGET, int(last["node"][p]), list(sh),
                     cap.masks_to_lists(last["alloc_mask"][p], len(sh)), int(last["uids"][p])))
    m.records(recs)
    # filter and bind on the owner
    bound = {}
    for r in range(g.world):
        own = g.own(r)
        if len(own) < 8:
            continue
        ids = np.sort(rng.choice(np.arange(own.start, own.stop), min(64, len(own)), replace=False)).astype(np.int32)
        sh = list(interned[int(rng.integers(0, len(interned)))])
        node = m.filter_bind(ids, sh, uid, rng)
        if node is not None:
            bound[uid] = node
            uid += 1
    return uid, bound


@pytest.mark.parametrize("world", STATE_WORLDS)
def test_state_across_batches_on_a_group(world):
    """One group, one twin, one oracle through six batches whose shape counts cross the 16 / 32 / 96 / host-formed
    geometries, with records, owner filter / bind, node reloads (one node per shard, and a bulk load across a shard
    boundary) and one restore between them.  After every batch: outputs, the rows of every shard and the caches of
    every shape interned so far, per shard on its owner."""
    rng = np.random.default_rng(500 + world)
    nodes = hetero_nodes(rng, 1200)
    cl = Cluster(1, nodes)
    o, twin = cl.oracle(), cl.handle()
    interned, uid, last, owner_bound = [], 1 << 40, None, {}
    with ShardGroup(cl, world) as g:
        m = _Mirror(g, twin, o, 1, nodes)
        for k, (n_old, n_new) in enumerate(STATE_PLAN):
            if last is not None:
                uid, bound = _between(m, rng, interned, last, uid)
                owner_bound.update(bound)
                if k == 2:                                       # one node per shard reloaded at a new size
                    for r in range(world):
                        own = g.own(r)
                        if len(own):
                            m.node_set(own[len(own) // 2], int(rng.choice([1, 2, 4, 8])), int(rng.choice([16384, 81920])))
                if k == 3:                                       # rows across the boundary of shards 0 and 1
                    lo = g.ranges[1][0]
                    core = rng.choice([100, 60, 0], (6, 2)).astype(np.int32)
                    mem = rng.integers(0, 40961, (6, 2)).astype(np.int32)
                    m.load_bulk(lo - 3, 2, 40960, core, mem)
                if k == 4:
                    m.restore()
                    owner_bound = {}
            old = [interned[int(i)] for i in rng.choice(len(interned), min(n_old, len(interned)), replace=False)] if interned else []
            new = mixed_shapes(rng, n_new, avoid=interned)
            shapes = old + new
            pick = pod_picks(rng, shapes, 1500, "trickle" if len(shapes) > 96 else "front")
            b = Batch(1, nodes, shapes, pick)
            uids = np.arange(uid, uid + b.n_pods, dtype=np.uint64); uid += b.n_pods
            ref = _run_group_batch(g, twin, m.o, b.c_off, b.units, uids=uids)
            interned += new
            check_shards(g, m.o, interned, sample_nodes(len(nodes), 400, k, ref["node"]))
            check_shards(g, m.o)                                 # rows of every node
            check_uids(g, m.o, uids[:: 7], owner_bound)
            last = dict(ref, uids=uids, shapes=[shapes[int(s)] for s in pick])
    twin.close()


# ------------------------------------------------------------------------------------------------ mutation streams
def _stream(g, rng, P, uid0):
    """Records for a batch of P pods: at pod 0, at pod P, several at one position, AddPods on a node of every shard,
    ForgetPods of pods the oracle placed earlier in the batch (filled in as the oracle runs)."""
    at = sorted([0, 0, P, P] + [int(x) for x in rng.integers(1, P, 10)] + [P // 2] * 3)
    adds = []
    for j, a in enumerate(at):
        r = j % g.world
        own = g.own(r)
        if not len(own):
            own = range(0, g.n_nodes)
        node = int(rng.integers(own.start, own.stop))
        adds.append((a, node, uid0 + j))
    return adds


def _oracle_segments(eg, o, w, adds, uids, rng):
    """The oracle runs the batch segment by segment, the records in between; a third of the records become ForgetPods
    of pods placed earlier in the same batch.  Returns (outputs, records, positions)."""
    cap = eg.capi
    ref = {f: [] for f in FIELDS}
    recs, mut_at, placed, prev = [], [], [], 0
    P = w.n_pods
    cuts = sorted(set(a for a, _, _ in adds))
    for cut in cuts + ([P] if P not in cuts else []):
        if cut > prev:
            seg = eg.workloads.window(w, prev, cut - prev)
            r = o.schedule_batch(seg.c_off, seg.units64(), uids=uids[prev:cut], threads=4)
            for f in FIELDS:
                ref[f].append(r[f])
            for i in np.nonzero(r["status"] == 0)[0]:
                req = [tuple(int(x) for x in seg.units[k]) for k in range(int(seg.c_off[i]), int(seg.c_off[i + 1]))]
                placed.append((int(uids[prev + i]), int(r["node"][i]), req, cap.masks_to_lists(r["alloc_mask"][i], len(req))))
            prev = cut
        for a, node, uid in [x for x in adds if x[0] == cut]:
            if placed and rng.integers(0, 3) == 0:
                u, n, req, alloc = placed.pop(int(rng.integers(0, len(placed))))
                rec = (cap.EGS_MUT_FORGET, n, req, alloc, u)
            else:
                rec = (cap.EGS_MUT_ADD, node, [(int(rng.choice([10, 25])), 2048, 0)], [[int(rng.integers(0, w.gpus))]], uid)
            oracle_mut(o, rec)
            recs.append(rec); mut_at.append(cut)
    return {f: np.concatenate(ref[f]) for f in FIELDS}, recs, mut_at


@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 7, 8])
def test_mutation_streams(world):
    """schedule_batch_mut on a group: records at pod 0, at pod P and repeated at one position, on nodes of every
    shard, first with explicit uids, then with library uids.  Outputs equal the oracle segment by segment; rows and
    caches per shard; pod_known / pod_released of the batch uids on every rank and of an owner-bound uid on the
    owner."""
    eg = egs()
    rng = np.random.default_rng(world)
    w = eg.workloads.config(2, n_nodes=1500, n_pods=3000)
    cl = Cluster.of_workload(w)
    o, twin = cl.oracle(), cl.handle()
    lib = LibUids()
    with ShardGroup(cl, world) as g:
        # a bind on the owner first: its uid lives in the owner's pod maps only
        node = w.n_nodes - 2
        req = [tuple(int(x) for x in w.units[0])]
        want = o.bind(node, req, 7)
        assert g.on_owner(node, lambda r, h: h.bind(node, req, 7)) == want and twin.bind(node, req, 7) == want
        for half, explicit in ((0, True), (1, False)):
            part = eg.workloads.window(w, half * 1500, 1500)
            if explicit:
                uids = np.arange(10_000 + half * 5000, 10_000 + half * 5000 + part.n_pods, dtype=np.uint64)
            else:
                uids = lib.take(part.n_pods)
            adds = _stream(g, rng, part.n_pods, 1_000_000 + half * 1000)
            ref, recs, mut_at = _oracle_segments(eg, o, part, adds, uids, rng)
            u = uids if explicit else None
            outs = g.each(lambda r, h: h.schedule_batch_mut(part.c_off, part.units, mut_at, recs, uids=u, mode=2))
            tw = twin.schedule_batch_mut(part.c_off, part.units, mut_at, recs, uids=u, mode=2)
            check_outputs(outs, ref, f"stream {half} ({'explicit' if explicit else 'library'} uids)", tw)
            check_shards(g, o, eg.workloads.shapes_of(part), sample_nodes(w.n_nodes, 400, half, ref["node"]))
            check_uids(g, o, list(uids[::5]) + [r[4] for r in recs], {7: node})


# ------------------------------------------------------------------------------------------------ back to back
def test_batches_back_to_back():
    """Each rank of a group of 6 runs four batches through one `seq`, with no join across ranks between them (the
    peers' copies of a rank's buffer from one batch's last round may still be in flight when its next batch starts).
    Every batch equals the twin's and the oracle's; then rows and caches per shard."""
    rng = np.random.default_rng(66)
    nodes = hetero_nodes(rng, 1500)
    cl = Cluster(0, nodes)
    o, twin = cl.oracle(), cl.handle()
    batches, all_shapes = [], []
    for n_shapes in (10, 30, 120, 20):
        shapes = mixed_shapes(rng, n_shapes, avoid=all_shapes)
        all_shapes += shapes
        batches.append(Batch(0, nodes, shapes, pod_picks(rng, shapes, 1200, "trickle" if n_shapes > 96 else "front")))
    lib = LibUids()
    refs = [o.schedule_batch(b.c_off, b.units.astype(np.int64), uids=lib.take(b.n_pods), threads=4) for b in batches]
    twins = [twin.schedule_batch(b.c_off, b.units, mode=2) for b in batches]
    with ShardGroup(cl, 6) as g:
        outs = g.seq([lambda r, h, b=b: h.schedule_batch(b.c_off, b.units, mode=2) for b in batches])
        for k in range(len(batches)):
            check_outputs([outs[r][k] for r in range(6)], refs[k], f"batch {k}", twins[k])
        check_shards(g, o, all_shapes, sample_nodes(len(nodes), 500, 66))
    twin.close()
