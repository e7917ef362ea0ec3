"""One handle's call stream, as the cgo extender sends it, on the C oracle: a seeded generator of steps -- Filter /
Score / Bind for one pod at a time, AddPod / ForgetPod / replay singly and as mutation records, node reloads, batches
through all five entry points, checkpoint what-ifs, headroom and eviction what-ifs -- and the oracle's answer to each.
A GPU test runs the same steps on a library handle and compares every answer (tests/test_gpu_call_stream.py).

The generator reads the oracle's state (GPU counts, podsMaps, placed pods), so it is deterministic per seed.  Every step
is a plain dict that replays on a fresh oracle to the same state: a checkpoint rollback, which the oracle cannot do, is
a fresh oracle that replays the steps up to the save.

A sub-stream owns the nodes n with n % parts == part and a uid range of its own, and only calls that touch nothing
else (no full node list, no library-assigned uids, no checkpoint); sub-streams of one cluster run on one handle from
concurrent threads and must each see what the oracle running them one after the other sees.

Importing this module loads neither libegs nor a GPU."""
from collections import Counter

import numpy as np

import evict_model as em
import headroom_model as hm
import oracle_c as oc

SENT = (-1, -1, 0)
OK, NOFIT, NO_OPTION, TRANSACT, BAD_ARG, PANIC = 0, 1, 2, 3, 4, 9
ADD, FORGET, REPLAY = 0, 1, 2
AUTO_UID0 = 1 << 63                                   # the first library-assigned uid of a handle
RESCAN, ROUNDS = 1, 2
MEMS = (16384, 40960, 81920)
RSMAX = 96                                            # distinct shapes one round set of the rounds engine holds
SHAPE_CACHE = 256                                     # shapes past which the handle rebuilds its shape cache

BASE = [
    [(50, 16384, 0)], [(25, 4096, 0)], [(0, 8192, 0)], [(10, 0, 0)],
    [(30, 8192, 0), (30, 8192, 0), (10, 2048, 0)], [(20, 4096, 0), (10, 2048, 0)],
    [(0, 0, 1)], [(0, 0, 2)], [(0, 0, 8)], [(0, 0, 1), SENT], [SENT, (25, 4096, 0)], [SENT],
    [(40, 8192, 0), (0, 0, 1), (20, 1024, 0), SENT],
]
GEOMETRY = {
    "8": dict(g_max=8, c_max=4, gpus=(1, 2, 4, 8), modes=(0, RESCAN, ROUNDS),
              base=BASE),
    "wide": dict(g_max=16, c_max=4, gpus=(4, 12, 16), modes=(0, RESCAN),
                 base=BASE + [[(0, 0, 12)], [(0, 0, 3), (10, 1024, 0)], [(0, 0, 16)]]),
    "sidecar": dict(g_max=8, c_max=8, gpus=(1, 2, 4, 8), modes=(0, RESCAN),
                    base=BASE + [[(20, 4096, 0), SENT, SENT, (0, 0, 1), (0, 0, 1)],
                                 [(0, 0, 1)] * 6 + [SENT, SENT],
                                 [(10, 1024, 0), (10, 1024, 0), SENT, (0, 0, 1), SENT, (0, 0, 1)],
                                 [(5, 512, 0), SENT, (5, 512, 0), SENT, (5, 512, 0)]]),   # 5 branches: leaf-split
}
# step kinds that change the scheduler state (a checkpoint save changes nothing observable)
MUTATING = ("filter", "filter_score", "score", "schedule_one", "bind", "apply", "replay", "cancel", "records", "reload", "load",
            "batch", "rollback")
READ_ONLY = ("peek", "headroom", "evict", "known", "save", "drop")
ENTRIES = ("plain", "nodes", "mut", "vec", "device")


def branches(req):
    """Containers Trade tries on every GPU (all but whole-GPU ones)."""
    return sum(1 for u in req if u[2] == 0)


def fresh_shape(k):
    """The k-th shape of the stream's own, each distinct from every other and from BASE."""
    c, m = 1 + k % 97, 128 * (1 + k // 97)
    r = k % 5
    if r == 3:
        return [(c, m, 0), (10, 1024, 0)]
    if r == 4:
        return [(0, 0, 1), (c, m, 0)]
    return [(c, m, 0)]


def mix64(x):
    """egs_mix64 of a uint64 array."""
    with np.errstate(over="ignore"):
        z = x.astype(np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def digests(ids, scores):
    """(fit digest, score digest) of a pod whose fit nodes are `ids` with `scores`."""
    ids = np.asarray(ids, np.uint64)
    s = (np.asarray(scores, np.int64) & 0xFFFFFFFF).astype(np.uint64)
    with np.errstate(over="ignore"):
        fd = mix64(2 * ids + np.uint64(1)).sum(dtype=np.uint64)
        sd = (mix64(2 * ids + np.uint64(2)) * (np.uint64(2) * s + np.uint64(1))).sum(dtype=np.uint64)
    return np.uint64(fd), np.uint64(sd)


def masks_of(alloc, planes):
    m = np.zeros(planes, np.uint16)
    for c, a in enumerate(alloc or []):
        m[c] = sum(1 << g for g in a)
    return m


def lists_of(masks, C):
    return [[g for g in range(16) if (int(masks[c]) >> g) & 1] for c in range(C)]


def c_off_units(reqs):
    c_off = np.concatenate([[0], np.cumsum([len(r) for r in reqs])]).astype(np.int32)
    units = np.array([u for r in reqs for u in r], np.int64).reshape(-1, 3)
    return c_off, units


# ------------------------------------------------------------------------------------------------ the oracle side
class Model:
    """The C oracle of one cluster and what the library's answers depend on beyond it: the shapes the handle has
    interned (a checkpoint rollback forgets later ones), the next library-assigned uid and the open checkpoint."""

    def __init__(self, policy, nodes, geo):
        g = GEOMETRY[geo]
        self.policy, self.geo, self.g_max, self.c_max = policy, geo, g["g_max"], g["c_max"]
        self.planes = 8 if self.c_max > 4 else 4
        self.nodes0 = nodes
        self.o = oc.OracleC(policy)
        self.G, self.mt = [], []
        for n, (gc, mt, rows) in enumerate(nodes):
            assert self.o.add_node(100 * gc, mt * gc) == n
            if rows is not None:
                self.o.set_rows(n, rows[0], rows[1])
            self.G.append(gc); self.mt.append(mt)
        self.N = len(nodes)
        self.interned = {}                               # shape tuple -> None, in interning order
        self.next_uid = AUTO_UID0
        self.ck = None                                   # (log length, interned) at the open checkpoint's save
        self.log = []                                    # the steps that made the current state

    def intern(self, req):
        self.interned.setdefault(tuple(tuple(u) for u in req), None)

    # ---- the reference's calls, as oracle_harness.oracle_batch drives them
    def filter(self, ids, req):
        return self.o.filter(ids, req)

    def one(self, ids, req, uid):
        """filter `ids` (None: every node), score the fit ones, bind the first maximal one."""
        fit = self.o.filter(ids, req)
        cand = np.arange(self.N, dtype=np.int32) if ids is None else np.asarray(ids, np.int32)
        fid = cand[fit.astype(bool)]
        if len(fid) == 0:
            return fit, fid, OK, np.zeros(0, np.int64), -1, NOFIT, None
        st, sc = self.o.score(fid, req)
        w = int(fid[int(np.argmax(sc))])
        bst, alloc = self.o.bind(w, req, uid)
        return fit, fid, st, sc, w, bst, alloc

    def record(self, rec):
        kind, node, req, alloc, uid = rec
        if kind == FORGET:
            return self.o.forget_pod(node, req, alloc, uid)
        if kind == REPLAY:
            return self.o.replay_pod(node, req, alloc, uid)
        return self.o.add_pod(node, req, alloc, uid)

    def batch(self, reqs, uids, cands=None, mut_at=(), recs=(), vec_pods=0):
        """The driver rule pod by pod (oracle_harness.oracle_batch) with the masks of every GPU and plane, the node
        list cands[p] of each pod (None: every node), records applied before pod mut_at[j] and the full fit / score
        vectors of the first vec_pods pods.  Returns the six outputs (+ vec_fit / vec_score) and each pod's GPU lists."""
        P, N = len(reqs), self.N
        out = dict(node=np.full(P, -1, np.int32), status=np.zeros(P, np.int32),
                   alloc_mask=np.zeros((P, self.planes), np.uint16), fit_count=np.zeros(P, np.int32),
                   fit_digest=np.zeros(P, np.uint64), score_digest=np.zeros(P, np.uint64))
        if vec_pods:
            out["vec_fit"] = np.zeros((vec_pods, N), np.uint8)
            out["vec_score"] = np.zeros((vec_pods, N), np.int64)
        allocs = [None] * P
        j = 0
        indexed = self.geo == "8" and cands is None and not vec_pods
        p = 0
        while p < P:
            while j < len(mut_at) and mut_at[j] == p:
                self.record(recs[j]); j += 1
            if indexed:                                  # pods [p, q) up to the next record through the C driver
                q = mut_at[j] if j < len(mut_at) else P
                c_off, units = c_off_units(reqs[p:q])
                r = self.o.schedule_batch_indexed(c_off, units, np.asarray(uids[p:q], np.uint64))
                for f in out:
                    out[f][p:q] = r[f]
                for k in range(p, q):
                    if r["status"][k - p] == OK:
                        allocs[k] = lists_of(r["alloc_mask"][k - p], len(reqs[k]))
                p = q
                continue
            req = reqs[p]
            ids = None if cands is None else cands[p]
            if ids is not None and len(ids) == 0:
                out["status"][p] = NOFIT
                p += 1
                continue
            fit, fid, st, sc, w, bst, alloc = self.one(ids, req, int(uids[p]))
            assert st == OK
            out["fit_count"][p] = len(fid)
            out["fit_digest"][p], out["score_digest"][p] = digests(fid, sc)
            out["node"][p], out["status"][p] = w, bst
            if p < vec_pods:
                out["vec_fit"][p] = fit
                out["vec_score"][p][fid] = sc
            if bst == OK:
                out["alloc_mask"][p] = masks_of(alloc, self.planes)
                allocs[p] = alloc
            p += 1
        while j < len(mut_at):
            self.record(recs[j]); j += 1
        return out, allocs

    def headroom(self, shapes, node0, n, node_set, limit):
        """headroom_model on every node of [node0, node0 + n) inside node_set (None: every node)."""
        S = len(shapes)
        count, failed, capped = np.zeros((S, n), np.int32), np.zeros((S, n), np.int32), np.zeros((S, n), bool)
        inside = None if node_set is None else set(int(x) for x in node_set)
        for s, req in enumerate(shapes):
            for i in range(n):
                nd = node0 + i
                if inside is not None and nd not in inside:
                    continue
                na = hm.allocator(self.o.rows(nd), self.mt[nd], self.policy, req, self.o.peek(nd, req))
                count[s, i], failed[s, i], capped[s, i] = hm.node_headroom(na, req, limit)
        summary = np.array([[int(count[s].sum()), int((count[s] > 0).sum()), int(failed[s].sum()),
                             int(capped[s].sum())] for s in range(S)], np.int64)
        return count, failed, summary

    def evict(self, req, ids, victims):
        """evict_model on each candidate: the victims its podsMap holds forgotten, then the pending pod."""
        st, sc, al = [], [], []
        for n, vs in zip(ids, victims):
            n = int(n)
            held = [v[2] for v in vs if self.o.node_has_pod(n, v[2])]
            na = hm.allocator(self.o.rows(n), self.mt[n], self.policy, req, self.o.peek(n, req))
            na.pods_map = dict.fromkeys(held, True)
            a, b, c = em.node_evict(na, req, em.applied(held, vs))
            st.append(a); sc.append(b); al.append(c)
        return np.array(st, np.int32), np.array(sc, np.int64), al

    # ---- one step
    def apply(self, step):
        """Run `step` on the oracle; returns the answer the library must give."""
        k = step["kind"]
        if k not in READ_ONLY:
            self.log.append(step)
        o = self.o
        if k == "filter":
            self.intern(step["req"])
            return dict(fit=self.filter(step["ids"], step["req"]))
        if k == "filter_score":
            self.intern(step["req"])
            fit = self.filter(step["ids"], step["req"])
            cand = np.arange(self.N, dtype=np.int32) if step["ids"] is None else np.asarray(step["ids"], np.int32)
            st, sc = o.score(cand[fit.astype(bool)], step["req"])
            return dict(fit=fit, status=st, score=sc)
        if k == "score":
            self.intern(step["req"])
            st, sc = o.score(step["ids"], step["req"])
            return dict(status=st, score=sc)
        if k == "schedule_one":
            self.intern(step["req"])
            fit, fid, st, sc, w, bst, alloc = self.one(step["ids"], step["req"], step["uid"])
            return dict(fit=fit, status=st, score=sc, node=w, bind=bst, alloc=alloc)
        if k == "bind":
            self.intern(step["req"])
            st, alloc = o.bind(step["node"], step["req"], step["uid"])
            return dict(status=st, alloc=alloc)
        if k == "peek":
            self.intern(step["req"])
            return dict(opt=[o.peek(n, step["req"]) for n in step["nodes"]])
        if k in ("apply", "replay", "cancel"):
            kind = dict(apply=ADD, replay=REPLAY, cancel=FORGET)[k]
            return dict(status=self.record((kind, step["node"], step["req"], step["alloc"], step["uid"])))
        if k == "records":
            for r in step["records"]:
                assert self.record(r) == OK
            return dict(status=OK)
        if k == "reload":
            n, G, mt = step["node"], step["gpus"], step["mt"]
            assert o.node_reset(n, 100 * G, mt * G) == 0
            self.G[n], self.mt[n] = G, mt
            return dict(status=OK)
        if k == "load":
            o.set_rows(step["node"], step["core"], step["mem"])
            return dict(status=OK)
        if k == "batch":
            reqs = step["reqs"]
            for r in reqs:
                self.intern(r)
            uids = step["uids"]
            if uids is None:
                uids = np.arange(self.next_uid, self.next_uid + len(reqs), dtype=np.uint64)
                self.next_uid += len(reqs)
            cands = None
            if step["sets"] is not None:
                cands = [np.asarray(step["sets"][s], np.int32) for s in step["pod_set"]]
            out, allocs = self.batch(reqs, uids, cands, step["mut_at"], step["records"], step["vec_pods"])
            out["uids"], out["allocs"] = uids, allocs
            return out
        if k == "headroom":
            for r in step["shapes"]:
                self.intern(r)
            count, failed, summary = self.headroom(step["shapes"], step["node0"], step["n"], step["set"],
                                                   step["limit"])
            return dict(count=count, failed=failed, summary=summary)
        if k == "evict":
            self.intern(step["req"])
            st, sc, al = self.evict(step["req"], step["ids"], step["victims"])
            return dict(status=st, score=sc, alloc=al)
        if k == "known":
            return dict(known=np.array([o.known_pod(u) for u in step["uids"]], bool),
                        released=np.array([o.released_pod(u) for u in step["uids"]], bool))
        if k == "save":
            self.ck = (len(self.log), dict(self.interned))
            return dict(status=OK)
        if k == "drop":
            self.ck = None
            return dict(status=OK)
        if k == "rollback":
            self.log.pop()
            self.fork()
            return dict(status=OK)
        raise ValueError(k)

    def fork(self):
        """Back to the open checkpoint: a fresh oracle replays the steps up to the save."""
        n_log, interned = self.ck
        log = self.log[:n_log]
        fresh = Model(self.policy, self.nodes0, self.geo)
        for s in log:
            fresh.apply(s)
        self.o, self.G, self.mt, self.next_uid, self.log = fresh.o, fresh.G, fresh.mt, fresh.next_uid, fresh.log
        self.interned = dict(interned)


# ------------------------------------------------------------------------------------------------ the generator
def cluster(rng, n, gpus, mems=MEMS):
    """n nodes [(gpu_count, mem_total per GPU, (core row, mem row) or None)]: a third fresh, the others partly used,
    empty or above their totals (headroom_cases.nodes); every id is set."""
    out = []
    for _ in range(n):
        g, mt = int(rng.choice(gpus)), int(rng.choice(mems))
        if rng.integers(0, 3) == 0:
            out.append((g, mt, None))
            continue
        core, mem = [], []
        for _ in range(g):
            k = rng.integers(0, 4)
            if k == 0:
                c, m = 100, mt
            elif k == 1:
                c, m = int(rng.choice([0, 10, 35, 60, 90])), int(rng.integers(0, mt + 1))
            elif k == 2:
                c, m = int(rng.integers(100, 140)), mt + int(rng.integers(0, mt // 4 + 3))
            else:
                c, m = 0, 0
            core.append(c); mem.append(m)
        out.append((g, mt, (core, mem)))
    return out


WEIGHTS = dict(filter=12, score=6, schedule_one=14, bind=4, peek=2, apply=5, replay=3, cancel=6, records=5,
               reload=2, load=2, batch=12, headroom=2, evict=4, known=3, whatif=4)


class Stream:
    """A seeded stream of steps on a cluster of n_nodes nodes of geometry `geo`.  part / parts: the sub-stream of one
    of `parts` concurrent callers.  steps: the stream's length, which paces its shapes so that more than 256 are
    interned past the middle, the first time under an open checkpoint (serial streams only)."""

    def __init__(self, seed, geo, policy, n_nodes, steps, part=0, parts=1, nodes=None, model=None,
                 big_batch=2000, weights=None, pace=True):
        self.seed, self.geo, self.steps = seed, geo, steps
        self.rng = np.random.default_rng(seed)
        g = GEOMETRY[geo]
        self.gpus, self.modes, self.base = g["gpus"], g["modes"], [list(s) for s in g["base"]]
        self.part, self.parts, self.serial = part, parts, parts == 1
        self.pace = pace and self.serial                 # the scripted crossings of 256 and of RSMAX shapes
        crng = np.random.default_rng(seed + 7919)
        self.model = model or Model(policy, nodes or cluster(crng, n_nodes, self.gpus), geo)
        m = self.model
        self.N = m.N
        self.own = np.arange(part, self.N, parts, dtype=np.int32)
        self.shapes = [list(s) for s in self.base]       # the shapes the stream has used
        self.n_fresh = 0
        self.uid = 1 + (part << 40) + (seed << 48)
        self.pool = []                                   # (node, req, alloc, uid) of pods placed by the stream
        self.pool_at_save = 0
        self.used_uids = []
        self.released_uids = []
        self.big_batch = big_batch
        w = dict(WEIGHTS, **(weights or {}))
        if not self.serial:
            w["whatif"] = 0
        self.kinds = [k for k in w if w[k] > 0]
        self.entries = [k for k in ("filter", "filter_score", "score", "schedule_one", "bind", "peek", "apply",
                                    "replay", "cancel", "records", "reload", "load", "headroom", "evict", "known")
                        if w.get(k if k != "filter_score" else "score", 0) > 0]
        self.entries += ["batch:" + x for x in (ENTRIES if self.serial else ("nodes",))] if w["batch"] else []
        self.p = np.array([w[k] for k in self.kinds], float)
        self.p /= self.p.sum()
        self.i = 0
        self.fresh_left = 3
        self.queue = []                                  # steps already decided (a what-if's save / rollback)
        self.ck_done = False                             # the scripted what-if across 256 shapes ran
        self.wide_done = False                           # the scripted batch of > RSMAX shapes ran
        self.last_batch_uids = []
        self.counts = Counter()
        self.statuses = Counter()
        self.after = set()                               # (last state-changing kind, kind)
        self.prev_mut = None
        self.max_interned = 0
        self.crossed_under_ck = False
        self.widest_batch = 0

    # ---- draws
    def r(self, n):
        return int(self.rng.integers(0, n))

    def new_uid(self):
        self.uid += 1
        self.used_uids.append(self.uid)
        return self.uid

    def target_shapes(self):
        """The shapes the stream aims to have interned by now: 240 by a fifth of its length, where the scripted
        what-if takes it past 256 under an open checkpoint, and 340 once that ran."""
        if not self.pace:
            return 40
        return 340 if self.ck_done else min(240, 20 + int(240 * self.i / max(1, 0.2 * self.steps)))

    def req(self, cheap=False, fresh_ok=True):
        """A request: a new shape (at most 3 per step) while the stream is below its pace, else a used one (half of
        them from BASE)."""
        m = self.model
        if fresh_ok and not cheap and self.fresh_left > 0 and len(m.interned) < self.target_shapes() and \
                self.rng.random() < 0.5:
            self.fresh_left -= 1
            return self.fresh()
        pool = self.base if self.rng.random() < 0.5 else self.shapes
        for _ in range(20):
            sh = pool[self.r(len(pool))]
            if not cheap or (branches(sh) <= 3 and len(sh) <= 4):
                return sh
        return [(25, 4096, 0)]

    def fresh(self):
        sh = fresh_shape(self.n_fresh + 4000 * self.part)
        self.n_fresh += 1
        self.shapes.append(sh)
        return sh

    def ids(self, k=None, dup=True):
        k = k or 1 + self.r(min(len(self.own), 400))
        ids = self.rng.choice(self.own, size=min(k, len(self.own)), replace=False).astype(np.int32)
        if dup and self.rng.random() < 0.2:
            ids = np.concatenate([ids, ids[self.rng.integers(0, len(ids), 1 + self.r(4))]])
            self.rng.shuffle(ids)
        return ids

    def node(self):
        return int(self.own[self.r(len(self.own))])

    def fits_record(self, node, alloc):
        return all(len(a) <= 8 and all(g < self.model.G[node] for g in a) for a in alloc)

    def pooled(self, recent=False, record=True):
        """A pod of the pool whose GPU lists still fit its node, recent ones first when `recent`."""
        if not self.pool:
            return None
        for _ in range(8):
            i = len(self.pool) - 1 - self.r(min(40, len(self.pool))) if recent else self.r(len(self.pool))
            node, req, alloc, uid = self.pool[i]
            if all(g < self.model.G[node] for a in alloc for g in a) and (not record or self.fits_record(node, alloc)):
                return self.pool[i]
        return None

    def synth(self, node, record=True):
        """A pod another scheduler placed on `node`: up to 8 containers, whole GPUs, sentinels, fractions."""
        G = self.model.G[node]
        req, alloc = [], []
        for _ in range(1 + self.r(8) if self.rng.random() < 0.3 else 1 + self.r(3)):
            k = self.r(4)
            if k == 0:
                cnt = 1 + self.r(min(G, 8 if record else 16))
                req.append((0, 0, cnt)); alloc.append(sorted(self.rng.choice(G, cnt, replace=False).tolist()))
            elif k == 1:
                req.append(SENT); alloc.append([self.r(G)])
            else:
                req.append((int(self.rng.choice([5, 10, 25, 40])), int(self.rng.choice([256, 1024, 4096])), 0))
                alloc.append([self.r(G)])
        return node, req, alloc, self.new_uid()

    def pod(self, record=True):
        p = self.pooled(recent=self.rng.random() < 0.5, record=record) if self.rng.random() < 0.7 else None
        return p or self.synth(self.node(), record)

    def records(self, k):
        out = []
        for _ in range(k):
            node, req, alloc, uid = self.pod()
            r = self.r(10)
            if r < 4:
                out.append((ADD, node, req, alloc, uid))
            elif r < 6:
                out.append((REPLAY, node, req, alloc, uid))
            elif r < 8:
                out.append((FORGET, node, req, alloc, uid))
            elif r == 8:
                out.append((FORGET, -1, req, alloc, uid))
            else:
                out.append((FORGET, node, req, alloc, self.new_uid()))       # a uid nobody holds
        return out

    def node_set(self):
        """A candidate set inside the stream's own nodes: dense, sparse or empty."""
        d = float(self.rng.choice([0.0, 0.02, 0.2, 0.6, 1.0]))
        keep = self.rng.random(len(self.own)) < d
        return np.sort(self.own[keep]).astype(np.int32)

    # ---- steps
    def next(self):
        """The next step (a dict), checked against the geometry, run on the oracle; returns (step, answer)."""
        self.fresh_left = 3
        step = self.queue.pop(0) if self.queue else self.draw()
        if step is None:                                 # a what-if's step, drawn when its turn comes
            step = self.draw(whatif=False)
        check_step(step, self.model)
        ref = self.model.apply(step)
        self.account(step, ref)
        self.i += 1
        return step, ref

    def draw(self, whatif=True):
        if whatif and self.pace and not self.ck_done and len(self.model.interned) >= 236:
            return self.whatif(scripted=True)
        if self.pace and not self.wide_done and len(self.shapes) > RSMAX + 30:
            self.wide_done = True
            reqs = [self.shapes[i] for i in self.rng.permutation(len(self.shapes))[:RSMAX + 24]]
            reqs = [r for r in reqs for _ in range(1 + self.r(3))]
            return self.batch("plain", reqs)
        if self.prev_mut is not None and (self.prev_mut == "rollback" or self.rng.random() < 0.3):
            # steer: an entry point that has not run yet after the last state-changing kind
            missing = [x for x in self.entries if (self.prev_mut, x) not in self.after]
            if missing:
                x = missing[self.r(len(missing))]
                if x.startswith("batch:"):
                    return self.batch(x[6:], [self.req() for _ in range(1 + self.r(8))])
                return getattr(self, "s_" + x)()
        k = self.kinds[int(self.rng.choice(len(self.kinds), p=self.p))]
        if k == "whatif":                                # early in the stream: a rollback replays the steps so far
            return self.whatif() if whatif and self.i < 0.12 * self.steps else self.draw(whatif)
        return getattr(self, "s_" + k)()

    def whatif(self, scripted=False):
        """save, k steps, rollback, sometimes a second what-if from the same save, then drop or keep the checkpoint.
        The scripted one interns shapes past 256 while the checkpoint is open."""
        k = 2 + self.r(12)
        seq = [dict(kind="save")]
        if scripted:
            self.ck_done = True
            reqs = [self.fresh() for _ in range(SHAPE_CACHE + 8 - len(self.model.interned))]
            seq.append(self.batch("plain", reqs + [self.shapes[self.r(len(self.shapes))] for _ in range(20)]))
        seq += [None] * k + [dict(kind="rollback")]
        if self.rng.random() < 0.3:
            seq += [None] * (1 + self.r(10)) + [dict(kind="rollback")]
        if self.rng.random() < 0.5:
            seq.append(dict(kind="drop"))
        self.queue = seq[1:]                             # None: a step drawn when its turn comes
        return seq[0]

    def s_filter(self):
        ids = None if self.serial and self.rng.random() < 0.3 else self.ids()
        return dict(kind="filter", ids=ids, req=self.req())

    def s_score(self):
        """Score over the nodes a filter of the same request just found fit (kube-scheduler's order), or over any
        nodes, some of them without an option (EGS_ERR_PANIC when one of those fits)."""
        if self.rng.random() < 0.6:
            return self.s_filter_score()
        return dict(kind="score", ids=self.ids(dup=False), req=self.req())   # Score is serial in the reference

    def s_filter_score(self):
        ids = None if self.serial and self.rng.random() < 0.3 else self.ids()
        return dict(kind="filter_score", ids=ids, req=self.req())

    def s_schedule_one(self):
        ids = None if self.serial and self.rng.random() < 0.4 else self.ids(dup=False)
        return dict(kind="schedule_one", ids=ids, req=self.req(), uid=self.new_uid())

    def s_bind(self):
        p = self.pooled(record=False) if self.rng.random() < 0.4 else None
        uid = p[3] if p is not None else self.new_uid()
        return dict(kind="bind", node=self.node(), req=self.req(fresh_ok=False), uid=uid)

    def s_peek(self):
        return dict(kind="peek", nodes=[self.node() for _ in range(1 + self.r(4))], req=self.req(fresh_ok=False))

    def _single(self, kind):
        node, req, alloc, uid = self.pod(record=False)
        if kind == "cancel":
            r = self.r(10)
            if r == 0:
                node = -1
            elif r == 1:
                uid = self.new_uid()
        return dict(kind=kind, node=node, req=req, alloc=alloc, uid=uid)

    def s_apply(self):
        return self._single("apply")

    def s_replay(self):
        return self._single("replay")

    def s_cancel(self):
        return self._single("cancel")

    def s_records(self):
        return dict(kind="records", records=self.records(1 + self.r(12)))

    def s_reload(self):
        n = self.node()
        held = [p for p in self.pool if p[0] == n]
        if held and self.rng.random() < 0.7:
            n = held[-1][0]
        G = self.model.G[n] if self.rng.random() < 0.5 else int(self.rng.choice(self.gpus))
        return dict(kind="reload", node=n, gpus=G, mt=int(self.rng.choice(MEMS)))

    def s_load(self):
        n = self.node()
        G, mt = self.model.G[n], self.model.mt[n]
        core = [int(self.rng.choice([0, 10, 35, 60, 90, 100, 120])) for _ in range(G)]
        mem = [int(self.rng.integers(0, mt + mt // 4 + 1)) for _ in range(G)]
        return dict(kind="load", node=n, core=core, mem=mem)

    def s_batch(self):
        entry = ENTRIES[self.r(5)] if self.serial else "nodes"
        r = self.rng.random()
        P = 1 + self.r(16) if r < 0.85 else 16 + self.r(80) if r < 0.99 else 96 + self.r(max(1, self.big_batch - 95))
        P = min(P, self.big_batch)
        if entry == "vec":
            P = min(P, 60)
        return self.batch(entry, [self.req() for _ in range(P)])

    def batch(self, entry, reqs):
        P = len(reqs)
        uids = None
        if entry != "device" and (not self.serial or self.rng.random() < 0.5):
            uids = np.array([self.new_uid() for _ in range(P)], np.uint64)
            self.last_batch_uids = uids.tolist()
        mode = 0 if entry in ("vec",) else int(self.rng.choice(self.modes))
        step = dict(kind="batch", entry=entry, mode=mode, reqs=reqs, uids=uids, sets=None, pod_set=None,
                    mut_at=(), records=(), vec_pods=0)
        if entry == "nodes":
            ns = 1 + self.r(3)
            step["sets"] = [self.node_set() for _ in range(ns)]
            if ns == 1 or self.rng.random() < 0.5:
                step["pod_set"] = np.sort(self.rng.integers(0, ns, P)).astype(np.int32)
            else:
                step["pod_set"] = self.rng.integers(0, ns, P).astype(np.int32)
        if entry == "mut":
            k = 1 + self.r(10)
            step["records"] = self.records(k)
            step["mut_at"] = np.sort(self.rng.integers(0, P + 1, k)).astype(np.int32)
        if entry == "vec":
            step["vec_pods"] = min(P, 1 + self.r(3))
        return step

    def s_headroom(self):
        shapes = [self.req(cheap=True) for _ in range(1 + self.r(2))]
        n = 1 + self.r(min(self.N, 120))
        node0 = self.r(self.N - n + 1)
        if self.serial:
            node_set = None if self.rng.random() < 0.5 else self.node_set()
        else:
            node_set = self.own
        return dict(kind="headroom", shapes=shapes, node0=node0, n=n, set=node_set, limit=1 + self.r(4))

    def s_evict(self):
        """Candidates in random order, half of the time led by the nodes of the latest placements, whose uids a batch
        may have left pending."""
        req = self.req(cheap=True)
        ids = self.ids(k=1 + self.r(min(40, len(self.own))), dup=False)
        if self.pool and self.rng.random() < 0.5:
            recent = list(dict.fromkeys(p[0] for p in reversed(self.pool[-30:])))[:1 + self.r(8)]
            ids = np.array(list(dict.fromkeys(recent + [int(x) for x in ids])), np.int32)
            self.rng.shuffle(ids)
        victims = [self.victims(int(n)) for n in ids]
        return dict(kind="evict", req=req, ids=ids, victims=victims)

    def victims(self, node):
        own = [p for p in self.pool[-400:] if p[0] == node and self.fits_record(node, p[2])]
        out = []
        for _ in range(self.r(6)):
            r = self.r(12)
            if own and r < 6:
                p = own[-1] if r < 3 else own[self.r(len(own))]
                out.append((p[1], p[2], p[3]))
            elif r == 6 and self.pool:
                out.append(([(10, 1024, 0)], [[0]], self.pool[self.r(len(self.pool))][3]))
            elif r == 7:
                out.append(([(0, 0, 1)], [[0]], self.new_uid()))
            elif r == 8 and self.released_uids:
                out.append(([(5, 512, 0)], [[0]], self.released_uids[self.r(len(self.released_uids))]))
            elif r >= 9 and out:
                out.append(out[self.r(len(out))])
        return out

    def s_known(self):
        k = 1 + self.r(20)
        uids = list(self.last_batch_uids[:k])
        if self.used_uids:
            uids += [self.used_uids[self.r(len(self.used_uids))] for _ in range(k)]
        uids += [AUTO_UID0 + self.r(64)] if self.serial else []
        return dict(kind="known", uids=[int(u) for u in uids])

    # ---- bookkeeping of what the stream reached
    def account(self, step, ref):
        m, k = self.model, step["kind"]
        self.counts[k if k != "batch" else "batch:" + step["entry"]] += 1
        if k == "batch":
            self.counts["batch"] += 1
        name = k if k != "batch" else "batch:" + step["entry"]
        if self.prev_mut is not None:
            self.after.add((self.prev_mut, name))
        if k in MUTATING:
            self.prev_mut = name
        for key in ("status", "bind"):
            v = ref.get(key) if isinstance(ref, dict) else None
            if v is None:
                continue
            for s in np.atleast_1d(v).tolist():
                self.statuses[int(s)] += 1
        if k == "save":
            self.pool_at_save = len(self.pool)
        elif k == "rollback":                            # the pods placed since the save never were
            del self.pool[self.pool_at_save:]
        n_int = len(m.interned)
        if n_int > SHAPE_CACHE and self.max_interned <= SHAPE_CACHE and m.ck is not None:
            self.crossed_under_ck = True
        self.max_interned = max(self.max_interned, n_int)
        if k == "batch":
            self.widest_batch = max(self.widest_batch, len({tuple(map(tuple, r)) for r in step["reqs"]}))
            for p, a in enumerate(ref["allocs"]):
                if a is not None:
                    self.pool.append((int(ref["node"][p]), step["reqs"][p], a, int(ref["uids"][p])))
        elif k in ("schedule_one", "bind") and ref.get("bind", ref.get("status")) == OK and ref.get("alloc"):
            node = ref["node"] if k == "schedule_one" else step["node"]
            self.pool.append((node, step["req"], ref["alloc"], step["uid"]))
        elif k in ("apply", "replay") and step["node"] >= 0:
            self.pool.append((step["node"], step["req"], step["alloc"], step["uid"]))
        elif k == "cancel" and m.o.released_pod(step["uid"]):
            self.released_uids.append(step["uid"])
        elif k == "records":
            self.released_uids += [r[4] for r in step["records"] if r[0] == FORGET and m.o.released_pod(r[4])]

    def report(self):
        return dict(steps=self.i, kinds=dict(self.counts), statuses=dict(self.statuses), max_shapes=self.max_interned,
                    shapes_past_256_under_checkpoint=self.crossed_under_ck, widest_batch=self.widest_batch,
                    pairs=len(self.after))


def check_step(step, m):
    """Every step is valid for the geometry of `m` in its state: shapes within c_max (8 for accounting), node ids
    set, GPU indices below the node's count, at most 8 per record container, modes the handle takes, batch uids
    distinct and unknown, sets inside the handle."""
    k = step["kind"]
    N = m.N

    def req_ok(req, cmax):
        assert 1 <= len(req) <= cmax, f"{k}: {len(req)} containers"
        for c, mm, cnt in req:
            assert cnt >= 0 and c >= -1 and mm >= -1, f"{k}: unit {(c, mm, cnt)}"

    def alloc_ok(node, req, alloc, record):
        assert len(alloc) == len(req)
        for a in alloc:
            assert all(0 <= g < m.G[node] for g in a), f"{k}: GPU index past node {node}'s {m.G[node]} GPUs"
            assert not record or len(a) <= 8, f"{k}: a record lists at most 8 GPUs"

    def ids_ok(ids):
        assert ids is None or (len(ids) == 0 or (min(ids) >= 0 and max(ids) < N))

    if k in ("filter", "score", "schedule_one", "filter_score"):
        req_ok(step["req"], m.c_max); ids_ok(step["ids"])
    elif k in ("bind", "peek"):
        req_ok(step["req"], m.c_max)
        ids_ok([step["node"]] if k == "bind" else step["nodes"])
    elif k in ("apply", "replay", "cancel"):
        req_ok(step["req"], 8)
        if step["node"] >= 0:
            alloc_ok(step["node"], step["req"], step["alloc"], False)
        else:
            assert k == "cancel"
    elif k == "records":
        for kind, node, req, alloc, uid in step["records"]:
            req_ok(req, 8)
            if node >= 0:
                alloc_ok(node, req, alloc, True)
            else:
                assert kind == FORGET
    elif k == "reload":
        assert 1 <= step["gpus"] <= m.g_max and step["gpus"] in GEOMETRY[m.geo]["gpus"]
    elif k == "load":
        G = m.G[step["node"]]
        assert len(step["core"]) == len(step["mem"]) == G
        assert all(0 <= x <= 1 << 20 for x in step["core"]) and all(0 <= x <= 1 << 25 for x in step["mem"])
    elif k == "batch":
        for r in step["reqs"]:
            req_ok(r, m.c_max)
        assert step["mode"] in GEOMETRY[m.geo]["modes"]
        if step["uids"] is not None:
            u = [int(x) for x in step["uids"]]
            assert len(set(u)) == len(u) and not any(m.o.known_pod(x) for x in u), "batch uids known or repeated"
        if step["sets"] is not None:
            assert 1 <= len(step["sets"]) <= 3
            for s in step["sets"]:
                ids_ok(s)
            assert all(0 <= x < len(step["sets"]) for x in step["pod_set"])
        assert list(step["mut_at"]) == sorted(step["mut_at"]) and all(0 <= x <= len(step["reqs"]) for x in step["mut_at"])
        for kind, node, req, alloc, uid in step["records"]:
            if node >= 0:
                alloc_ok(node, req, alloc, True)
        assert step["entry"] != "device" or step["uids"] is None
    elif k == "headroom":
        for r in step["shapes"]:
            req_ok(r, m.c_max)
            assert branches(r) <= 3
        assert 0 <= step["node0"] and step["node0"] + step["n"] <= N and 1 <= step["limit"] <= 1 << 18
    elif k == "evict":
        req_ok(step["req"], m.c_max)
        assert len(set(int(x) for x in step["ids"])) == len(step["ids"])
        for n, vs in zip(step["ids"], step["victims"]):
            for u, a, uid in vs:
                alloc_ok(int(n), u, a, True)


def diff(ref, got):
    """None when the library's answer `got` equals the oracle's `ref`, else the first field that differs."""
    for key, a in ref.items():
        if key in ("uids", "allocs"):
            continue
        b = got[key]
        if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
            a, b = np.asarray(a), np.asarray(b)
            if a.shape != b.shape:
                return f"{key}: shape {b.shape}, the oracle's {a.shape}"
            bad = np.argwhere(a != b)
            if bad.size:
                i = tuple(bad[0])
                return f"{key}[{', '.join(map(str, i))}] = {b[i]}, the oracle has {a[i]}"
        elif a != b:
            return f"{key} = {b}, the oracle has {a}"
    return None
