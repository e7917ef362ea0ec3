"""The call-stream harness (tests/call_stream.py) without a GPU: the generator is deterministic per seed and emits only
steps valid for its geometry; a checkpoint rollback (a fresh oracle replaying the steps up to the save) gives back the
state at the save; the headroom and eviction expectations read from the C oracle equal the Python mirror
(oracle/egs_oracle.py) running the same stream; and egso_node_has_pod agrees with the mirror's podsMaps."""
import numpy as np
import pytest

import call_stream as cs
import egs_oracle as po
import evict_model as em
import headroom_model as hm


def canon(x):
    """A step or an answer as plain Python values, for equality."""
    if isinstance(x, dict):
        return {k: canon(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [canon(v) for v in x]
    if isinstance(x, np.ndarray):
        return x.tolist()
    if isinstance(x, np.generic):
        return x.item()
    return x


@pytest.mark.parametrize("geo", ["8", "wide", "sidecar"])
def test_deterministic_per_seed(geo):
    a, b, c = (cs.Stream(seed, geo, 0, 67, 300) for seed in (5, 5, 6))
    ra = [canon(a.next()) for _ in range(300)]
    assert ra == [canon(b.next()) for _ in range(300)]
    assert ra != [canon(c.next()) for _ in range(300)]


@pytest.mark.parametrize("geo", ["8", "wide", "sidecar"])
def test_steps_valid_for_the_geometry(geo):
    """Stream.next checks every step (check_step) against the oracle state it is drawn from; a sub-stream stays
    inside its node partition and uid range and makes no call that touches anything else."""
    s = cs.Stream(7, geo, 1, 90, 1500)
    for _ in range(1500):
        s.next()
    assert s.max_interned > cs.SHAPE_CACHE and s.crossed_under_ck and s.widest_batch > cs.RSMAX
    assert all(s.counts[k] > 0 for k in s.entries)
    parts = 3
    subs = [cs.Stream(8, geo, 0, 90, 300, part=0, parts=parts)]
    subs += [cs.Stream(8 + t, geo, 0, 90, 300, part=t, parts=parts, model=subs[0].model) for t in (1, 2)]
    for t, sub in enumerate(subs):
        lo = 1 + (t << 40) + (sub.seed << 48)
        for _ in range(300):
            step, _ = sub.next()
            k = step["kind"]
            assert k not in ("save", "rollback", "drop") and (k != "batch" or step["entry"] == "nodes")
            nodes = [step[x] for x in ("node",) if x in step] + list(step.get("nodes") or [])
            assert step.get("ids", 0) is not None and step.get("set", 0) is not None, k
            nodes += list(step.get("ids") if step.get("ids") is not None else [])
            nodes += [r[1] for r in step.get("records", ())]
            nodes += [x for st in (step.get("sets") or []) for x in st]
            assert all(n % parts == t for n in nodes if n >= 0), (k, nodes)
            uids = [step["uid"]] if "uid" in step else []
            uids += list(step.get("uids") if step.get("uids") is not None else [])
            uids += [r[4] for r in step.get("records", ())] + [v[2] for vs in step.get("victims", ()) for v in vs]
            assert all(lo <= int(u) < lo + (1 << 40) for u in uids), k


def _state(m, uids):
    ids = np.arange(m.N, dtype=np.int32)
    rows = m.o.rows_many(ids, 16)
    caches = [m.o.peek_many(ids, list(sh), m.planes) for sh in m.interned]
    caches = [(p, np.where(p, s, 0), np.where(p[:, None], a, 0)) for p, s, a in caches]
    pods = [[m.o.node_has_pod(n, u) for n in range(m.N)] for u in uids]
    return canon([rows, caches, [m.o.known_pod(u) for u in uids], [m.o.released_pod(u) for u in uids], pods,
                  m.next_uid, sorted(m.interned)])


def test_rollback_replay_gives_the_state_at_the_save():
    s = cs.Stream(9, "8", 0, 70, 1200)
    seen = 0
    saved = None
    for _ in range(1200):
        nxt = s.queue[0] if s.queue else None
        if nxt is not None and nxt.get("kind") == "rollback":
            s.next()
            assert _state(s.model, uids) == saved, "the fork differs from the state at the save"
            seen += 1
            continue
        step, _ = s.next()
        if step["kind"] == "save":
            uids = list(s.used_uids)
            saved = _state(s.model, uids)
    assert seen >= 2


# ------------------------------------------------------------------------------------------------ the Python mirror
class Mirror:
    """The stream on egs_oracle.Scheduler: the steps that change state, and headroom / evict answered from the
    mirror's own NodeAllocators."""

    def __init__(self, policy, nodes):
        self.s = po.Scheduler(policy)
        for g, mt, rows in nodes:
            self.s.add_node(100 * g, mt * g)
            if rows is not None:
                self.s.set_rows(len(self.s.nodes) - 1, rows[0], rows[1])
        self.policy, self.next_uid = policy, cs.AUTO_UID0

    def assume(self, ids, req):
        return [1 if self.s.nodes[n].assume(req) is not None else 0 for n in ids]

    def one(self, ids, req, uid):
        fid = [n for n, f in zip(ids, self.assume(ids, req)) if f]
        if fid:
            sc = self.s.score(fid, req)
            self.s.bind(fid[sc.index(max(sc))], req, uid)

    def record(self, kind, node, req, alloc, uid):
        req, alloc = [tuple(u) for u in req], [list(a) for a in alloc]
        if kind == cs.FORGET:
            self.s.forget_pod(node, req, alloc, uid)
        elif kind == cs.REPLAY:
            self.s.nodes[node].add(uid, po.GPUOption(request=req, allocated=alloc))
        else:
            self.s.add_pod(node, req, alloc, uid)

    def apply(self, step):
        k, N = step["kind"], len(self.s.nodes)
        req = [tuple(u) for u in step.get("req") or []]
        ids = list(range(N)) if step.get("ids") is None else [int(x) for x in step["ids"]]
        if k == "filter":
            self.assume(ids, req)
        elif k == "filter_score":
            fid = [n for n, f in zip(ids, self.assume(ids, req)) if f]
            self.s.score(fid, req)
        elif k == "score":                            # Assume of a node without an entry, then the panic
            for n in ids:
                na = self.s.nodes[n]
                if na.key(req) not in na.allocated:
                    na.assume(req)
        elif k == "schedule_one":
            self.one(ids, req, step["uid"])
        elif k == "bind":
            self.s.bind(step["node"], req, step["uid"])
        elif k in ("apply", "replay", "cancel"):
            self.record(dict(apply=cs.ADD, replay=cs.REPLAY, cancel=cs.FORGET)[k], step["node"], req, step["alloc"],
                        step["uid"])
        elif k == "records":
            for r in step["records"]:
                self.record(*r)
        elif k == "reload":
            G, mt = step["gpus"], step["mt"]
            self.s.nodes[step["node"]] = po.NodeAllocator.new(100 * G, mt * G, self.policy)
        elif k == "load":
            self.s.set_rows(step["node"], step["core"], step["mem"])
        elif k == "batch":
            P = len(step["reqs"])
            uids = step["uids"]
            if uids is None:
                uids = [self.next_uid + p for p in range(P)]
                self.next_uid += P
            recs = list(zip(step["mut_at"], step["records"]))
            for p, r in enumerate(step["reqs"]):
                while recs and recs[0][0] == p:
                    self.record(*recs.pop(0)[1])
                cand = list(range(N)) if step["sets"] is None else [int(x) for x in step["sets"][step["pod_set"][p]]]
                self.one(cand, [tuple(u) for u in r], int(uids[p]))
            for _, rec in recs:
                self.record(*rec)

    def headroom(self, step):
        out = []
        inside = None if step["set"] is None else set(int(x) for x in step["set"])
        for sh in step["shapes"]:
            sh = [tuple(u) for u in sh]
            out.append([hm.node_headroom(self.s.nodes[n], sh, step["limit"])[:2]
                        if inside is None or n in inside else (0, 0)
                        for n in range(step["node0"], step["node0"] + step["n"])])
        return out

    def evict(self, step):
        req = [tuple(u) for u in step["req"]]
        out = []
        for n, vs in zip(step["ids"], step["victims"]):
            na = self.s.nodes[int(n)]
            st, sc, al = em.node_evict(na, req, em.applied(na.pods_map, vs))
            out.append((st, sc, al))
        return out


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("geo", ["8", "wide"])
def test_headroom_and_evict_match_the_python_mirror(geo, policy):
    w = dict(cs.WEIGHTS, headroom=8, evict=10, whatif=0, peek=0, known=0)
    s = cs.Stream(21 + policy, geo, policy, 48, 700, weights=w, big_batch=60, pace=False)
    mirror = Mirror(policy, s.model.nodes0)
    checked = 0
    for i in range(700):
        step, ref = s.next()
        if step["kind"] == "headroom":
            want = mirror.headroom(step)
            got = [list(zip(c.tolist(), f.tolist())) for c, f in zip(ref["count"], ref["failed"])]
            assert got == [[tuple(x) for x in sh] for sh in want], f"step {i}: headroom"
            checked += 1
        elif step["kind"] == "evict":
            want = mirror.evict(step)
            got = list(zip(ref["status"].tolist(), ref["score"].tolist(), ref["alloc"]))
            assert canon(got) == canon(want), f"step {i}: evict"
            checked += 1
        else:
            mirror.apply(step)
        if step["kind"] not in cs.READ_ONLY and i % 50 == 0:
            assert [s.model.o.rows(n) for n in range(s.N)] == [mirror.s.rows(n) for n in range(s.N)], f"step {i}"
    assert checked > 50
    # egso_node_has_pod against the mirror's podsMaps, for every uid the stream used, on every node
    for u in s.used_uids:
        for n in range(s.N):
            assert s.model.o.node_has_pod(n, u) == (u in mirror.s.nodes[n].pods_map), (u, n)
