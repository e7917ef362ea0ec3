"""The leaf-split Trade of a sidecar handle at sizes where every CTA of k_trade_leaves reduces items of several
misses (tests/sidecar_cases.py), the probe and the commit span several blocks, miss lists pass 256 entries and id
lists pass the handle's padded node count; batches through every entry point with mutation records woven in; and
node ids that were never set, on every handle geometry.  Sizes follow the device's SM count, each test asserts the
geometry it relies on, and everything is compared with the C oracle (oracle_harness)."""
import os

import numpy as np
import pytest

from oracle_harness import FIELDS, Cluster, compare_caches, compare_outputs, compare_rows, egs, oracle_batch, \
    oracle_mut
from sidecar_cases import DFS, PLANTED, S5, S6, S8, SENT, SMALL, batch, batch_cluster, planted_cluster, \
    planted_nodes, pods, s8_count, several_items_per_cta

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 4
PROBE = PASS = 256                   # threads per block of k_trade_probe / k_trade_commit and of k_pass


@pytest.fixture(scope="module")
def n_sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pair(policy, nodes, g_max=8, c_max=8):
    cl = Cluster(policy, nodes, g_max, c_max=c_max)
    return cl.handle(), cl.oracle()


def _n_pad(max_nodes):
    return -(-max_nodes // 1024) * 1024


# ------------------------------------------------------------------------------------------------ verbs
@pytest.mark.parametrize("policy", [0, 1])
def test_verbs_on_planted_clusters(n_sm, policy):
    """Cold filter of S5 and S6 over every node, peek on every planted node, option_dump against peek_many; then bind
    a few planted winners, check that exactly they lost their option, and Trade again.  S8 (2^24 leaves per node) over
    an id list of planted nodes."""
    N = planted_nodes(n_sm)
    nodes, where = planted_cluster(N)
    e, o = _pair(policy, nodes)
    assert N > 256 and -(-N // PROBE) >= 2
    planted = np.unique(np.concatenate([where[k] for k in PLANTED]))
    uid = 1
    for sh in (S5, S6):
        req = list(sh)
        assert several_items_per_cta(N, sh, n_sm)                  # every node is a miss of this cold shape
        got, ref = e.filter(None, req), o.filter(None, req, threads=THREADS)
        bad = np.flatnonzero(got != ref)
        assert bad.size == 0, f"{sh}: filter differs on nodes {bad[:5].tolist()}"
        assert ref.any() and not ref.all()
        for i in planted:
            assert e.peek(int(i), req) == o.peek(int(i), req), f"{sh}: node {i}"
        compare_caches(e, o, [sh], range(N), unfit_check=True)
        fit = [int(where[k][j]) for k in ("late", "tie_tile", "tie_chunk", "tie_lane", "prefix", "absent5", "absent6",
                                          "absent7", "late_low") for j in (0, -1) if ref[where[k][j]]]
        assert len(fit) >= 6
        before = e.option_dump(req)[0].copy()
        for i in fit:
            assert e.bind(i, req, uid) == o.bind(i, req, uid)
            uid += 1
        st = e.option_dump(req)[0]
        assert sorted(np.flatnonzero(st != before).tolist()) == sorted(fit) and (st[fit] == 0).all()
        compare_rows(e, o, range(N))
        got, ref = e.filter(None, req), o.filter(None, req, threads=THREADS)
        assert np.array_equal(got, ref), f"{sh}: filter after the binds"
        compare_caches(e, o, [sh], range(N), unfit_check=True)
    k8 = s8_count(n_sm)
    ids = np.unique(np.concatenate([where[k][:1] for k in ("late", "tie_tile", "unfit_first", "prefix", "absent7")]
                                   + [where["early"][:k8], where["late_low"][:k8]])).astype(np.int32)
    assert several_items_per_cta(len(ids), S8, n_sm)
    got, ref = e.filter(ids, list(S8)), o.filter(ids, list(S8), threads=THREADS)
    assert np.array_equal(got, ref) and ref.any() and not ref.all()
    compare_caches(e, o, [S8], ids, unfit_check=True)
    for i in ids[ref.astype(bool)][:3]:
        assert e.bind(int(i), list(S8), uid) == o.bind(int(i), list(S8), uid)
        uid += 1
    compare_rows(e, o, ids)


# ------------------------------------------------------------------------------------------------ id lists
@pytest.mark.parametrize("policy", [0, 1])
def test_id_lists(n_sm, policy):
    """Filter over a list longer than the padded node count, with duplicates and ids -1, max_nodes and 2^30 (the miss,
    key and id buffers grow), then a shorter list; score over lists whose absent, fitting nodes lie in several probe
    and commit blocks (the reference's panic, with its scores), and over one whose absent nodes all fail to fit."""
    cap = egs().capi
    N = planted_nodes(n_sm)
    nodes, where = planted_cluster(N)
    e, o = _pair(policy, nodes)
    rng = np.random.default_rng(policy)
    L = _n_pad(N) + 700
    ids = np.concatenate([rng.permutation(N), rng.integers(0, N, L - N)]).astype(np.int32)
    ids[rng.integers(0, L, 6)] = [-1, N, 1 << 30, -1, N, 1 << 30]
    assert several_items_per_cta(N, S6, n_sm)
    got, ref = e.filter(ids, list(S6)), o.filter(ids, list(S6))       # one oracle worker: ids repeat
    bad = np.flatnonzero(got != ref)
    assert bad.size == 0, f"filter differs at ids {ids[bad[:5]].tolist()}"
    short = rng.permutation(N)[:700].astype(np.int32)
    got, ref = e.filter(short, list(S5)), o.filter(short, list(S5))
    assert np.array_equal(got, ref) and ref.any()
    compare_caches(e, o, [S5, S6], range(N), unfit_check=True)

    for sh in (S5, S6):
        e, o = _pair(policy, nodes)
        req = list(sh)
        half = np.arange(0, N, 3, dtype=np.int32)                     # a third of the nodes filtered first
        assert np.array_equal(e.filter(half, req), o.filter(half, req))
        allids = rng.permutation(N).astype(np.int32)
        absent_fit = np.setdiff1d(np.arange(N), half)[o.trade_fits(np.setdiff1d(np.arange(N), half), req)]
        assert len(np.unique(absent_fit // PROBE)) >= 2
        st_o, sc_o = o.score(allids, req)
        st_e, sc_e = e.score(allids, req)
        assert st_e == st_o == cap.EGS_ERR_PANIC
        assert np.array_equal(sc_e, sc_o)
        compare_caches(e, o, [sh], range(N), unfit_check=True)
        e, o = _pair(policy, nodes)
        unfit = where["unfit_first"]
        rest = np.setdiff1d(np.arange(N), unfit).astype(np.int32)
        assert np.array_equal(e.filter(rest, req), o.filter(rest, req))
        st_o, sc_o = o.score(np.arange(N, dtype=np.int32), req)
        st_e, sc_e = e.score(np.arange(N, dtype=np.int32), req)
        assert st_e == st_o == cap.EGS_OK and np.array_equal(sc_e, sc_o)


# ------------------------------------------------------------------------------------------------ batches
def _device_batch(e, c_off, units):
    import torch
    P = len(c_off) - 1
    t = dict(node=torch.zeros(P, dtype=torch.int32, device="cuda"), status=torch.zeros(P, dtype=torch.int32, device="cuda"),
             alloc_mask=torch.zeros(P * 8, dtype=torch.uint8, device="cuda"),
             fit_count=torch.zeros(P, dtype=torch.int32, device="cuda"),
             fit_digest=torch.zeros(P, dtype=torch.int64, device="cuda"),
             score_digest=torch.zeros(P, dtype=torch.int64, device="cuda"))
    e.schedule_batch_device(c_off, units, [t[f].data_ptr() for f in FIELDS])
    torch.cuda.synchronize()
    got = {f: t[f].cpu().numpy() for f in FIELDS}
    got["alloc_mask"] = got["alloc_mask"].reshape(P, 8)
    got["fit_digest"] = got["fit_digest"].view(np.uint64)
    got["score_digest"] = got["score_digest"].view(np.uint64)
    return got


BATCH_NODES = 1100


@pytest.mark.parametrize("policy", [0, 1])
def test_batches_through_every_entry_point(policy):
    """Leaf-split and DFS pods on a sidecar cluster of 1 100 nodes (k_pass: 5 blocks, best-score ties between nodes of
    the second and fourth block), cold and then warm on the same handle, through schedule_batch, schedule_batch_vec,
    schedule_batch_device and schedule_batch_nodes with node sets of two densities."""
    nodes, champ = batch_cluster(BATCH_NODES, 20 + policy)
    assert -(-BATCH_NODES // PASS) >= 4 and len(champ) >= 2
    rng = np.random.default_rng(policy)
    b1, b2 = batch(pods(rng, 48)), batch(pods(rng, 40))
    u1, u2 = np.arange(48, dtype=np.uint64) + 1000, np.arange(40, dtype=np.uint64) + 2000
    o = Cluster(policy, nodes).oracle()
    refs = [oracle_batch(o, *b1, u1, planes=8), oracle_batch(o, *b2, u2, planes=8)]
    assert (refs[0]["status"] == 0).sum() > 20
    sets = [rng.random(BATCH_NODES) < 0.3, rng.random(BATCH_NODES) < 0.85]
    os_ = Cluster(policy, nodes).oracle()
    prefs = []
    for (c_off, units), u in ((b1, u1), (b2, u2)):
        ps = np.arange(len(c_off) - 1) % 2
        prefs.append(oracle_batch(os_, c_off, units, u, node_ids=[np.flatnonzero(sets[s]) for s in ps], planes=8))
    for call in ("batch", "vec", "device", "nodes"):
        e = Cluster(policy, nodes, c_max=8).handle()
        for k, ((c_off, units), u) in enumerate(((b1, u1), (b2, u2))):
            if call == "batch":
                got = e.schedule_batch(c_off, units, uids=u)
            elif call == "vec":
                got = e.schedule_batch_vec(c_off, units, 3, uids=u)
            elif call == "device":
                got = _device_batch(e, c_off, units)
            else:
                got = e.schedule_batch_nodes(c_off, units, sets, pod_set=np.arange(len(c_off) - 1) % 2, uids=u)
            compare_outputs(prefs[k] if call == "nodes" else refs[k], got, f"{call}, batch {k}")
            if call == "batch" and k == 1:
                compare_rows(e, o, range(BATCH_NODES))
                compare_caches(e, o, [S5, S6] + DFS[:2], range(BATCH_NODES), unfit_check=True)
        e.close()


def _record(rng, o, n_nodes, kind, uid, bound, stale_shape):
    """One mutation record, applied to the oracle: ADD / REPLAY of 1..8 containers on a random node, ForgetPod of a
    pod this batch bound, or an AddPod on the node with the best cached option of a leaf-split shape, on its
    container 0's GPU, so that the next pod of that shape meets a stale option."""
    cap = egs().capi
    if kind == "forget" and bound:
        u, node, req, alloc = bound.pop(int(rng.integers(0, len(bound))))
        rec = (cap.EGS_MUT_FORGET, node, req, alloc, u)
    elif kind == "stale" and o.peek_many(range(n_nodes), list(stale_shape), 8)[0].any():
        present, score, masks = o.peek_many(range(n_nodes), list(stale_shape), 8)
        node = int(np.flatnonzero(present)[np.argmax(score[present])])
        g = int(masks[node, 0]).bit_length() - 1
        rec = (cap.EGS_MUT_ADD, node, [(1, 20, 0)], [[g]], uid)
    else:
        node = int(rng.integers(0, n_nodes))
        gc = o.gpu_count(node)
        pool = [(int(rng.integers(1, 30)), int(rng.integers(1, 8)), 0), SENT, (0, 0, 1)]
        req = [pool[int(rng.integers(0, 3))] for _ in range(int(rng.integers(1, 9)))]
        alloc = [[int(rng.integers(0, gc))] for _ in req]
        rec = (cap.EGS_MUT_ADD if kind == "add" else cap.EGS_MUT_REPLAY, node, req, alloc, uid)
    oracle_mut(o, rec)
    return rec


@pytest.mark.parametrize("policy", [0, 1])
def test_mutation_stream_in_a_sidecar_batch(policy):
    """schedule_batch_mut (per-pod engine) with a record after about every tenth pod: ADD / REPLAY of 1..8 containers,
    ForgetPods of pods this batch bound (all 8 masks back to index lists), and AddPods on the best cached leaf-split
    option, so that a later bind fails in Transact exactly where the oracle's does."""
    cap = egs().capi
    nodes, _ = batch_cluster(BATCH_NODES, 30 + policy)
    rng = np.random.default_rng(40 + policy)
    pl = pods(rng, 120, split_every=3)
    c_off, units = batch(pl)
    P = len(pl)
    uids = np.arange(P, dtype=np.uint64) + 1
    o = Cluster(policy, nodes).oracle()
    cuts = list(range(9, P, 10))
    kinds = ["stale", "add", "forget", "replay", "stale", "forget"]
    recs, mut_at, bound, segs, prev = [], [], [], [], 0
    for q, cut in enumerate(cuts + [P]):
        seg = oracle_batch(o, c_off[prev:cut + 1] - c_off[prev], units[c_off[prev]:c_off[cut]], uids[prev:cut], planes=8)
        segs.append(seg)
        for i in np.flatnonzero(seg["status"] == 0):
            req = pl[prev + i]
            bound.append((int(uids[prev + i]), int(seg["node"][i]), req, cap.masks_to_lists(seg["alloc_mask"][i], len(req))))
        prev = cut
        if cut == P:
            break
        stale = next((pl[p] for p in range(cut, P) if pl[p] in (list(S5), list(S6))), S6)
        recs.append(_record(rng, o, BATCH_NODES, kinds[q % len(kinds)], 10_000 + q, bound, stale))
        mut_at.append(cut)
    ref = {f: np.concatenate([s[f] for s in segs]) for f in FIELDS}
    assert (ref["status"] == cap.EGS_ERR_TRANSACT).any()
    assert any(r[0] == cap.EGS_MUT_FORGET and len(r[2]) >= 5 for r in recs)
    e = Cluster(policy, nodes, c_max=8).handle()
    got = e.schedule_batch_mut(c_off, units, mut_at, recs, uids=uids, mode=cap.EGS_MODE_RESCAN)
    compare_outputs(ref, got, "batch with mutations")
    compare_rows(e, o, range(BATCH_NODES))
    compare_caches(e, o, [S5, S6], range(BATCH_NODES), unfit_check=True)


# ------------------------------------------------------------------------------------------------ never-set ids
GEOMETRIES = {"default-rescan": (8, 4, 1), "default-rounds": (8, 4, 2), "wide": (16, 4, 1), "sidecar": (8, 8, 1)}


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("geometry", list(GEOMETRIES))
def test_never_set_ids(geometry, policy):
    """max_nodes about 1.5x the set nodes, with holes at id 0, at the last id and in every 256-node block: a hole never
    fits, never counts in a digest and never caches an option; once a node joins a hole between batches, the next
    batch schedules onto it (an 8-GPU whole-node pod fits nothing else)."""
    g_max, c_max, mode = GEOMETRIES[geometry]
    N = 900
    rng = np.random.default_rng(50 + policy)
    holes = np.unique(np.concatenate([[0, N - 1], np.arange(0, N, 256) + 100, rng.choice(N, 290, replace=False)]))
    nodes = []
    for i in range(N):
        if i in set(holes.tolist()):
            nodes.append(None)
            continue
        core = rng.choice([100, 100, 60, 30, 0], 8)
        mem = np.where(core == 100, 32, rng.choice([20, 12, 4, 0], 8))
        core[1], mem[1] = 60, 12                                    # no set node is all free
        nodes.append((8, 32, (core.tolist(), mem.tolist())))
    set_ids = np.array([i for i in range(N) if nodes[i] is not None], np.int32)
    assert len(holes) > N // 4 and len(set(holes // 256)) == -(-N // 256)
    shapes = SMALL + ([((20, 6, 0), SENT, (0, 0, 1))] if c_max == 4 else [S5, S6, DFS[0], DFS[2]])
    cl = Cluster(policy, nodes, g_max, c_max=c_max)
    e, o = cl.handle(), cl.oracle()
    pl = [list(shapes[p % len(shapes)]) for p in range(40)]
    c_off, units = batch(pl)
    ref = oracle_batch(o, c_off, units, np.arange(40) + 1, node_ids=[set_ids] * 40, planes=e.n_masks)
    got = e.schedule_batch(c_off, units, uids=np.arange(40, dtype=np.uint64) + 1, mode=mode)
    compare_outputs(ref, got, f"{geometry}, holes")
    assert (ref["status"] == 0).sum() > 10
    for sh in shapes:
        st = e.option_dump(list(sh))[0]
        assert (st[holes] != 1).all(), f"{sh}: a never-set id holds an option"
    compare_rows(e, o, set_ids)
    compare_caches(e, o, shapes, set_ids, unfit_check=True)
    joined = [int(holes[0]), int(holes[len(holes) // 2])]
    for h in joined:
        assert e.node_set(h, 8, 32) == 0
        assert o.node_reset(h, 800, 256) == 0
    ids = np.sort(np.concatenate([set_ids, joined])).astype(np.int32)
    pl2 = [[(0, 0, 8)], [(0, 0, 8)]] + pl[:12]
    c2, u2 = batch(pl2)
    ref = oracle_batch(o, c2, u2, np.arange(len(pl2)) + 100, node_ids=[ids] * len(pl2), planes=e.n_masks)
    got = e.schedule_batch(c2, u2, uids=np.arange(len(pl2), dtype=np.uint64) + 100, mode=mode)
    compare_outputs(ref, got, f"{geometry}, after a node joined")
    assert got["node"][0] == joined[0] and got["status"][0] == 0
    assert got["node"][1] == joined[1] and got["status"][1] == 0
