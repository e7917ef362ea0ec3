"""egs_evict_fit on the GPU, pinned by its two equalities (include/egs.h):
  A. per node, the checkpoint sequence -- save, egs_pod_cancel of each victim, filter / score / bind of the pending
     pod on that node alone, rollback -- gives the call's status, score and masks;
  B. for all candidates at once, save, egs_mutations_apply of every victim, a one-pod egs_schedule_batch_nodes over the
     candidate set, rollback, gives the batch outputs derived from the call's outputs.
Clusters carry a history (headroom_cases): a batch, then AddPod records that make cached options stale, then ForgetPod
records that release some pods.  Victims are drawn from the history's placements, with uids in another node's podsMap,
unknown and released uids, repeats, empty lists and whole-GPU pods.  The call must change nothing observable, refuse
every malformed argument without a change, and on a shard group answer for each rank's own nodes."""
import numpy as np
import pytest

import egs_oracle as po
import headroom_cases as hc
from oracle_harness import Cluster, egs
from shard_groups import ShardGroup

pytestmark = pytest.mark.gpu

RESCAN, ROUNDS = 1, 2
OK, NOFIT, TRANSACT = 0, 1, 3
SENT = hc.SENT
MEMS = (16384, 40960, 81920)
M64 = (1 << 64) - 1

SHAPES = [
    [(50, 16384, 0)], [(25, 4096, 0)], [(0, 8192, 0)],                       # single fractional, core 0 included
    [(30, 8192, 0), (30, 8192, 0), (10, 2048, 0)], [(20, 4096, 0), (10, 2048, 0)],   # multi-container
    [(0, 0, 1)], [(0, 0, 2)], [(0, 0, 8)],                                     # whole GPUs
    [(0, 0, 1), SENT], [SENT, (25, 4096, 0)],                                  # GPU + sentinel
]
WIDE_SHAPES = SHAPES + [[(0, 0, 12)], [(0, 0, 3), (10, 1024, 0)]]
SIDECAR_SHAPES = SHAPES + [
    [(20, 4096, 0), SENT, SENT, (0, 0, 1), (0, 0, 1)],
    [(0, 0, 1)] * 6 + [SENT, SENT],
    [(10, 1024, 0), (10, 1024, 0), SENT, SENT, (0, 0, 1)],
]
GEOMETRY = {"8": dict(g_max=8, c_max=4, gpus=(1, 2, 4, 8), shapes=SHAPES),
            "wide": dict(g_max=16, c_max=4, gpus=(4, 12, 16), shapes=WIDE_SHAPES),
            "sidecar": dict(g_max=8, c_max=8, gpus=(1, 2, 4, 8), shapes=SIDECAR_SHAPES)}


# ------------------------------------------------------------------------------------------------ clusters
class History:
    """A cluster on a handle after a history, and the pods its podsMaps hold: pool[node] = [(units, alloc, uid)]."""

    def __init__(self, seed, n, geo, policy=0, mode=RESCAN, n_pods=None):
        g = GEOMETRY[geo]
        self.rng = rng = np.random.default_rng(seed)
        self.cl = Cluster(policy, hc.nodes(rng, n, g["gpus"], MEMS), g["g_max"], g["c_max"])
        self.shapes = g["shapes"]
        c_off, units, uids, mut_at, recs = hc.history(rng, self.cl.nodes, self.shapes, n_pods or n, n // 5)
        self.batch = (c_off, units, uids, mut_at, recs)
        self.e = self.cl.handle()
        self.pool = {}
        self._collect(self.e.schedule_batch_mut(c_off, units, mut_at, recs, uids, mode=mode))

    def _collect(self, out):
        cap = egs().capi
        c_off, units, uids, _, recs = self.batch
        for p in np.nonzero(out["status"] == OK)[0]:
            req = [tuple(int(x) for x in units[k]) for k in range(c_off[p], c_off[p + 1])]
            alloc = cap.masks_to_lists(out["alloc_mask"][p], len(req))
            if max(len(a) for a in alloc) <= cap.EGS_MAX_GPUS:      # what a record can carry
                self.pool.setdefault(int(out["node"][p]), []).append((req, alloc, int(uids[p])))
        for _, node, req, alloc, uid in recs:
            self.pool.setdefault(node, []).append((req, alloc, uid))
        # some pods leave for good: their uids are released and their podsMap entries gone
        self.released, self.forgets = [], []
        for node in sorted(self.pool):
            if self.rng.random() < 0.05:
                req, alloc, uid = self.pool[node].pop(0) if self.pool[node] else (None, None, None)
                if uid is not None:
                    self.forgets.append((1, node, req, alloc, uid)); self.released.append(uid)
        self.apply_forgets(self.e)

    def apply_forgets(self, e):
        assert e.mutations_apply(self.forgets) == 0

    def victims(self, node):
        """A victim list for `node`: its own pods, a pod of another node's podsMap, unknown and released uids,
        repeats, or nothing."""
        rng, own = self.rng, self.pool.get(node, [])
        out = []
        for _ in range(int(rng.integers(0, 6))):
            r = int(rng.integers(0, 12))
            if own and r < 6:
                out.append(own[int(rng.integers(len(own)))])
            elif r == 6:
                other = self.pool[int(rng.choice(list(self.pool)))]
                if other:
                    out.append(([(10, 1024, 0)], [[0]], other[0][2]))
            elif r == 7:
                out.append(([(0, 0, 1)], [[0]], 10**12 + int(rng.integers(10**6))))
            elif r == 8 and self.released:
                out.append(([(5, 512, 0)], [[0]], int(rng.choice(self.released))))
            elif r >= 9 and out:
                out.append(out[int(rng.integers(len(out)))])
        return out

    def candidates(self, k):
        """k distinct nodes in random order, half of them (where there are enough) nodes the AddPod records touched,
        whose cached options may be stale."""
        touched = self.rng.permutation(sorted({r[1] for r in self.batch[4]}))[:k // 2]
        rest = self.rng.permutation(np.setdiff1d(np.arange(self.cl.n_nodes), touched))[:k - len(touched)]
        return self.rng.permutation(np.concatenate([touched, rest])).astype(np.int32)


# ------------------------------------------------------------------------------------------------ the equalities
def equality_a(e, req, ids, victims, status, score, masks, what):
    cap = egs().capi
    seen = set()
    for i, n in enumerate(ids.tolist()):
        e.checkpoint_save()
        try:
            for u, a, uid in victims[i]:
                assert e.pod_cancel(n, u, a, uid) == OK
            fit = int(e.filter([n], req)[0])
            st, sc = e.score([n], req)
            assert st == OK, what
            assert (fit == 0) == (status[i] == NOFIT), f"{what}: node {n} fit {fit}, status {status[i]}"
            assert sc[0] == score[i], f"{what}: node {n} score {sc[0]} != {score[i]}"
            if fit:
                bst, lists = e.bind(n, req, 1 << 62)
                assert bst == status[i], f"{what}: node {n} bind {bst} != {status[i]}"
                if bst == OK:
                    assert lists == cap.masks_to_lists(masks[i], len(req)), f"{what}: node {n} masks"
            if status[i] != OK:
                assert not masks[i].any(), f"{what}: node {n} masks of a failed bind"
            seen.add(int(status[i]))
        finally:
            e.checkpoint_rollback()
    return seen


def batch_of(ids, status, score, masks):
    """The six outputs of a one-pod batch over the candidate set, from the call's per-node outputs."""
    fit = status != NOFIT
    fd = sd = 0
    for n, s in zip(ids[fit].tolist(), score[fit].tolist()):
        fd = (fd + po.mix64(2 * n + 1)) & M64
        sd = (sd + po.mix64(2 * n + 2) * (2 * s + 1)) & M64
    if not fit.any():
        return dict(node=-1, status=NOFIT, alloc_mask=np.zeros_like(masks[0]), fit_count=0, fit_digest=0, score_digest=0)
    best = score[fit].max()
    w = int(ids[fit & (score == best)].min())
    i = int(np.nonzero(ids == w)[0][0])
    return dict(node=w, status=int(status[i]), alloc_mask=masks[i], fit_count=int(fit.sum()), fit_digest=fd,
                score_digest=sd)


def equality_b(e, req, ids, victims, mode, what):
    status, score, masks = e.evict_fit(req, ids, victims)
    recs = [(1, int(n), u, a, uid) for n, vs in zip(ids.tolist(), victims) for u, a, uid in vs]
    e.checkpoint_save()
    try:
        assert e.mutations_apply(recs) == OK
        c_off, units = hc.identical(req, 1)
        out = e.schedule_batch_nodes(c_off, units, [np.sort(ids)], mode=mode)
    finally:
        e.checkpoint_rollback()
    want = batch_of(ids, status, score, masks)
    for f, v in want.items():
        assert np.array_equal(out[f][0], v), f"{what}: {f} {out[f][0]} != {v}"
    return status


# ------------------------------------------------------------------------------------------------ 1. equality A
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("geo", ["8", "wide", "sidecar"])
def test_equality_a(geo, policy):
    h = History(100 + policy, 3000, geo, policy=policy, mode=ROUNDS if geo == "8" else RESCAN)
    seen, n_victims = set(), 0
    for s, req in enumerate(h.shapes):
        ids = h.candidates(250)
        victims = [h.victims(int(n)) for n in ids]
        n_victims += sum(map(len, victims))
        status, score, masks = h.e.evict_fit(req, ids, victims)
        seen |= equality_a(h.e, req, ids, victims, status, score, masks, f"{geo}, policy {policy}, shape {req}")
    assert seen == {OK, NOFIT, TRANSACT}, seen
    assert n_victims > 0


def test_equality_a_without_victims():
    """victim_off NULL: "filter, then bind status" on the current rows."""
    h = History(110, 2000, "8", mode=ROUNDS)
    for req in h.shapes[:4]:
        ids = h.candidates(300)
        status, score, masks = h.e.evict_fit(req, ids)
        equality_a(h.e, req, ids, [[]] * len(ids), status, score, masks, f"no victims, shape {req}")


# ------------------------------------------------------------------------------------------------ 2. equality B
@pytest.mark.parametrize("geo,mode", [("8", ROUNDS), ("8", RESCAN), ("wide", RESCAN), ("sidecar", RESCAN)])
def test_equality_b(geo, mode):
    h = History(200 + mode, 20_000, geo, mode=ROUNDS if geo == "8" else RESCAN)
    fits = 0
    for req in h.shapes[:3] + h.shapes[5:7] + h.shapes[-1:]:
        ids = h.candidates(4000)
        victims = [h.victims(int(n)) for n in ids]
        status = equality_b(h.e, req, ids, victims, mode, f"{geo}, mode {mode}, shape {req}")
        fits += int((status != NOFIT).sum())
    assert fits > 0


# ------------------------------------------------------------------------------------------------ 3. read-only
def _state(e, shapes, uids):
    dumps = [e.state_dump()] + [e.option_dump(list(sh)) for sh in shapes]
    return dumps, [e.pod_known(int(u)) for u in uids], [e.pod_released(int(u)) for u in uids]


def _same(a, b, what):
    (da, ka, ra), (db, kb, rb) = a, b
    for x, y in zip(da, db):
        for p, q in zip(x, y):
            assert np.array_equal(p, q), what
    assert ka == kb and ra == rb, what


def test_read_only():
    a = History(300, 3000, "8", mode=ROUNDS)
    b = History(300, 3000, "8", mode=ROUNDS)
    unseen = [(35, 12345, 0)]
    ids = a.candidates(2000)
    victims = [a.victims(int(n)) for n in ids]
    uids = sorted({v[2] for vs in victims for v in vs})
    before = _state(a.e, a.shapes, uids)
    for req in a.shapes + [unseen]:
        a.e.evict_fit(req, ids, victims)
    _same(before, _state(a.e, a.shapes, uids), "evict_fit changed the state")
    st, _, _ = a.e.option_dump(unseen)
    assert (st == 0).all()
    rng = np.random.default_rng(301)
    c_off, units = hc.pods(a.shapes, rng.integers(0, len(a.shapes), 3000))
    ra, rb = a.e.schedule_batch(c_off, units), b.e.schedule_batch(c_off, units)
    for f in ra:
        assert np.array_equal(ra[f], rb[f]), f"the batch after evict_fit differs in {f}"
    _same(_state(a.e, a.shapes, uids), _state(b.e, a.shapes, uids), "states after the batch differ")
    # with a checkpoint open
    a.e.checkpoint_save()
    saved = _state(a.e, a.shapes, uids)
    a.e.evict_fit([(45, 777, 0)], ids, victims)
    a.e.schedule_batch(c_off, units)
    a.e.checkpoint_rollback()
    _same(saved, _state(a.e, a.shapes, uids), "rollback after evict_fit")


# ------------------------------------------------------------------------------------------------ 4. refusals
def test_refusals():
    cap = egs().capi
    h = History(400, 1000, "8", mode=ROUNDS)
    e, L, p = h.e, h.e.L, cap._p
    unset = Cluster(0, [(2, 16384, None), None, (4, 16384, None)]).handle()
    req = cap.units_array([(25, 4096, 0)])
    ids = h.candidates(20)
    victims = [h.victims(int(n)) for n in ids]
    n0 = int(ids[0]); g0 = h.cl.nodes[n0][0]
    st_ = np.zeros(64, np.int32); sc = np.zeros(64, np.int32); am = np.zeros((64, 4), np.uint8)
    uids = sorted({v[2] for vs in victims for v in vs})
    before = _state(e, h.shapes, uids)

    def call(handle=e, C_=1, u=req, n=None, node_ids=ids, off=None, recs=None, outs=(st_, sc, am), vict=victims):
        node_ids = np.ascontiguousarray(node_ids, np.int32)
        n = len(node_ids) if n is None else n
        if off is None and vict is not None:
            off = np.concatenate([[0], np.cumsum([len(v) for v in vict])]).astype(np.int32)
            recs = cap.mutations_array([(1, int(nd), a, b, c) for nd, vs in zip(node_ids.tolist(), vict) for a, b, c in vs])
        return L.egs_evict_fit(handle.h, C_, p(u), n, p(node_ids), p(off), p(recs), *[p(x) for x in outs])

    assert call() == OK

    def with_record(kind=1, node=n0, units=((10, 1024, 0),), alloc=((0,),), n_idx=None):
        a = cap.mutations_array([(kind, node, list(units), [list(x) for x in alloc], 5)])
        if n_idx is not None:
            a[0]["n_idx"][0] = n_idx
        return call(node_ids=[n0], off=np.array([0, 1], np.int32), recs=a, vict=None)
    cases = dict(
        negative_n=call(n=-1), no_status=call(outs=(None, sc, am)), no_masks=call(outs=(st_, sc, None)),
        node_below=call(node_ids=[n0, -1], vict=None), node_past=call(node_ids=[h.cl.n_nodes], vict=None),
        repeated=call(node_ids=[n0, n0], vict=None),
        off_start=call(node_ids=[n0], off=np.array([1, 1], np.int32), recs=cap.mutations_array([]), vict=None),
        off_down=call(node_ids=[n0, int(ids[1])], off=np.array([0, 1, 0], np.int32),
                      recs=cap.mutations_array([(1, n0, [(10, 1024, 0)], [[0]], 5)]), vict=None),
        no_records=call(node_ids=[n0], off=np.array([0, 1], np.int32), recs=None, vict=None),
        add_record=with_record(kind=0), other_node=with_record(node=int(ids[1])),
        bad_unit=with_record(units=((0, 0, -1),)), nine_indices=with_record(n_idx=9),
        index_past=with_record(alloc=((g0,),)),
    )
    for what, rc in cases.items():
        assert rc == cap.EGS_ERR_BAD_ARG, f"{what}: {rc}"
        assert L.egs_last_error(e.h), what
    assert call(handle=unset, node_ids=[1], vict=None) == cap.EGS_ERR_NO_NODE
    # a malformed pending unit: what egs_filter returns for it
    for bad in ([(25, 4096, 0)] * 5, [(-2, 0, 0)], [(101 << 20, 0, 0)]):
        u = cap.units_array(bad)
        want = L.egs_filter(e.h, 1, p(np.array([n0], np.int32)), len(bad), p(u), p(np.zeros(1, np.uint8)))
        assert want != OK and call(C_=len(bad), u=u) == want, bad
    _same(before, _state(e, h.shapes, uids), "a refused call changed the state")
    # the leaf-split Trade of a sidecar handle is not served; a shape of 2^12 leaves is
    s = History(401, 200, "sidecar").e
    with pytest.raises(cap.EgsError) as ex:
        s.evict_fit([SENT] * 5, [0, 1])
    assert ex.value.status == cap.EGS_ERR_BAD_ARG and b"leaf-split" in s.L.egs_last_error(s.h)
    stt, _, _ = s.evict_fit([SENT] * 4, [0, 1])
    assert (stt == OK).all()
    # nothing to answer
    stt, _, _ = e.evict_fit(req.tolist(), [])
    assert len(stt) == 0


# ------------------------------------------------------------------------------------------------ 5. sharded
@pytest.mark.parametrize("world", [2, 4])
def test_sharded(world):
    cap = egs().capi
    h = History(500 + world, 4000, "8", mode=ROUNDS)
    c_off, units, uids, mut_at, recs = h.batch
    ids = h.candidates(1500)
    victims = [h.victims(int(n)) for n in ids]
    ref = [h.e.evict_fit(req, ids, victims) for req in h.shapes]
    with ShardGroup(h.cl, world) as g:
        g.each(lambda r, e: e.schedule_batch_mut(c_off, units, mut_at, recs, uids, mode=ROUNDS))
        g.each(lambda r, e: h.apply_forgets(e))

        def own(r, e):
            lo, hi = g.ranges[r]
            mine = (ids >= lo) & (ids < hi)
            vs = [v for v, m in zip(victims, mine) if m]
            for req, (st_, sc, am) in zip(h.shapes, ref):
                got = e.evict_fit(req, ids[mine], vs)
                assert np.array_equal(got[0], st_[mine]) and np.array_equal(got[1], sc[mine])
                assert np.array_equal(got[2], am[mine])
            other = int(ids[~mine][0])
            with pytest.raises(cap.EgsError) as ex:
                e.evict_fit(h.shapes[0], [other])
            assert ex.value.status == cap.EGS_ERR_BAD_ARG
            return True
        assert all(g.each(own))
