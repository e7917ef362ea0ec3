"""egs_headroom on the GPU, pinned by its definition: for every shape, the per-node counts equal a dry run
(checkpoint_save, schedule_batch of sum + 1 000 identical pods, checkpoint_rollback) on the same handle, node by node,
and the call changes nothing observable.  Clusters carry a history (headroom_cases): a batch, then AddPod records
that make cached options stale, on nodes partly used or above their totals."""
import numpy as np
import pytest

import headroom_cases as hc
from oracle_harness import Cluster, egs
from shard_groups import ShardGroup

pytestmark = pytest.mark.gpu

RESCAN, ROUNDS = 1, 2
SENT = hc.SENT
MEMS = (16384, 40960, 81920)


def cfg_shapes(cfg):
    w = egs().workloads
    return [list(sh) for sh in w.shapes_of(w.config(cfg, n_nodes=1, n_pods=4000))]


def mix():
    """config 4's 16 single fractional shapes (core 0 included), four of config 3's multi-container shapes, whole
    GPUs of count 1 / 2 / 8, and GPU + sentinel pods."""
    return cfg_shapes(4) + cfg_shapes(3)[:4] + [[(0, 0, 1)], [(0, 0, 2)], [(0, 0, 8)], [(0, 0, 1), SENT],
                                                [SENT, (25, 4096, 0)]]


def small_mix():
    """The shapes of mix() whose dry runs stay short enough for the per-pod engine on 10 000 nodes."""
    return [[(50, 40960, 0)], [(25, 40960, 0)], cfg_shapes(3)[1], cfg_shapes(3)[8], [(0, 0, 1)], [(0, 0, 2)],
            [(0, 0, 8)], [(0, 0, 1), SENT]]


def with_history(seed, n, shapes, mode, gpus=(1, 2, 4, 8), g_max=8, c_max=4, policy=0, n_pods=None):
    """A cluster of n nodes on a handle after a history of n_pods (default n) pods of `shapes`."""
    rng = np.random.default_rng(seed)
    cl = Cluster(policy, hc.nodes(rng, n, gpus, MEMS), g_max, c_max)
    e = cl.handle()
    c_off, units, uids, mut_at, recs = hc.history(rng, cl.nodes, shapes, n_pods or n, n // 5)
    e.schedule_batch_mut(c_off, units, mut_at, recs, uids, mode=mode)
    return cl, e, uids


def dry_run(e, sh, total, mode, node_set=None):
    c_off, units = hc.identical(sh, total + 1000)
    e.checkpoint_save()
    try:
        if node_set is None:
            return e.schedule_batch(c_off, units, mode=mode)
        return e.schedule_batch_nodes(c_off, units, [node_set], mode=mode)
    finally:
        e.checkpoint_rollback()


def check_against_dry_runs(e, shapes, mode, what, node_set=None):
    count, failed, summary = e.headroom(shapes, node_set=node_set)
    n_failed = 0
    for s, sh in enumerate(shapes):
        assert summary[s].tolist() == hc.summary_of(count[s], failed[s]), f"{what}: summary of shape {sh}"
        out = dry_run(e, sh, int(summary[s, 0] + summary[s, 2]), mode, node_set)
        hc.check_dry_run(count[s], failed[s], out, what=f"{what}, shape {sh}")
        n_failed += int(summary[s, 2])
    return count, failed, summary, n_failed


# ------------------------------------------------------------------------------------------------ 1. the dry run
@pytest.mark.parametrize("policy", [0, 1])
def test_equals_dry_run_rounds(policy):
    shapes = mix()
    _, e, _ = with_history(10 + policy, 10_000, shapes, ROUNDS, policy=policy)
    count, _, summary, n_failed = check_against_dry_runs(e, shapes, ROUNDS, f"rounds, policy {policy}")
    assert n_failed > 0, "no stale cached option failed its Transact"
    assert (summary[:, 0] > 0).all()


def test_equals_dry_run_rescan():
    shapes = small_mix()
    _, e, _ = with_history(20, 10_000, mix(), RESCAN, n_pods=30_000)
    check_against_dry_runs(e, shapes, RESCAN, "rescan")


def test_equals_dry_run_wide():
    shapes = small_mix() + [[(0, 0, 16)], [(0, 0, 3), (10, 1024, 0)]]
    _, e, _ = with_history(30, 10_000, small_mix(), RESCAN, gpus=(4, 12, 16), g_max=16)
    _, _, summary, _ = check_against_dry_runs(e, shapes, RESCAN, "wide")
    assert summary[-2, 0] > 0, "no 16-GPU node took a 16-GPU pod"


SIDECAR_SHAPES = [
    [(20, 4096, 0), SENT, SENT, (0, 0, 1), (0, 0, 1)],
    [(0, 0, 1)] * 6 + [SENT, SENT],
    [(10, 1024, 0), (10, 1024, 0), SENT, SENT, (0, 0, 1)],
    [(0, 0, 2), (25, 4096, 0), SENT, (0, 0, 1), SENT, (0, 0, 1), (0, 0, 1), SENT],
    [(50, 16384, 0)], [(0, 0, 1), SENT],
]


def test_equals_dry_run_sidecar():
    _, e, _ = with_history(40, 10_000, SIDECAR_SHAPES, RESCAN, c_max=8, n_pods=5000)
    _, _, summary, _ = check_against_dry_runs(e, SIDECAR_SHAPES, RESCAN, "sidecar")
    assert (summary[:4, 0] > 0).all()


def test_equals_dry_run_config4_size():
    eg = egs()
    w = eg.workloads.config(4, n_pods=500_000)
    e = Cluster.of_workload(w).handle()
    e.schedule_batch(w.c_off, w.units, mode=ROUNDS)
    sh = [(50, 40960, 0)]
    count, failed, summary = e.headroom([sh])
    out = dry_run(e, sh, int(summary[0, 0] + summary[0, 2]), ROUNDS)
    hc.check_dry_run(count[0], failed[0], out, what="config 4")
    assert summary[0].tolist() == hc.summary_of(count[0], failed[0]) and summary[0, 0] > 0


# ------------------------------------------------------------------------------------------------ 2. nothing changes
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
    shapes = mix()
    unseen = [(35, 12345, 0)]
    rng = np.random.default_rng(50)
    _, a, uids = with_history(50, 2000, shapes, ROUNDS)
    _, b, _ = with_history(50, 2000, shapes, ROUNDS)
    sample = rng.choice(uids, 200, replace=False).tolist() + [0x8000000000000000]
    before = _state(a, shapes, sample)
    a.headroom(shapes + [unseen])
    _same(before, _state(a, shapes, sample), "headroom changed the state")
    st, _, _ = a.option_dump(unseen)
    assert (st == 0).all()
    c_off, units = hc.pods(shapes, rng.integers(0, len(shapes), 3000))
    ra, rb = a.schedule_batch(c_off, units), b.schedule_batch(c_off, units)
    for f in ra:
        assert np.array_equal(ra[f], rb[f]), f"the batch after headroom differs in {f}"
    _same(_state(a, shapes, sample), _state(b, shapes, sample), "states after the batch differ")
    # with a checkpoint open
    a.checkpoint_save()
    saved = _state(a, shapes, sample)
    a.headroom(shapes + [[(45, 777, 0)]])
    a.schedule_batch(c_off, units)
    a.checkpoint_rollback()
    _same(saved, _state(a, shapes, sample), "rollback after headroom")


# ------------------------------------------------------------------------------------------------ 3. node sets
@pytest.mark.parametrize("mode", [RESCAN, ROUNDS])
def test_node_sets(mode):
    shapes = small_mix()
    cl, e, _ = with_history(60 + mode, 3000, mix(), mode)
    node_set = np.random.default_rng(mode).random(cl.n_nodes) < 0.5
    count, failed, _, _ = check_against_dry_runs(e, shapes, mode, f"node set, mode {mode}", node_set)
    assert not count[:, ~node_set].any() and not failed[:, ~node_set].any()
    full, _, _ = e.headroom(shapes)
    assert np.array_equal(count[:, node_set], full[:, node_set])


# ------------------------------------------------------------------------------------------------ 4. limit
def test_limit():
    shapes = small_mix()
    cl, e, _ = with_history(70, 3000, mix(), ROUNDS)
    node_set = np.random.default_rng(70).random(cl.n_nodes) < 0.7
    for zero in ([(0, 0, 0)], [SENT], [SENT, SENT]):
        count, failed, summary = e.headroom([zero], node_set=node_set, limit=37)
        assert (count[0, node_set] == 37).all() and not count[0, ~node_set].any() and not failed.any()
        assert summary[0].tolist() == [37 * int(node_set.sum()), int(node_set.sum()), 0, int(node_set.sum())]
    count, failed, _ = e.headroom(shapes)
    binds = count + failed
    for limit in (1, 2, 5):
        c, f, s = e.headroom(shapes, limit=limit)
        assert np.array_equal(c + f, np.minimum(binds, limit))
        assert np.array_equal(f, np.minimum(failed, limit))          # a failed bind is the first bind
        assert s[:, 3].tolist() == (binds > limit).sum(1).tolist()


# ------------------------------------------------------------------------------------------------ 5. sharded
@pytest.mark.parametrize("world", [2, 4])
def test_sharded(world):
    cap = egs().capi
    shapes = mix()
    rng = np.random.default_rng(80 + world)
    cl = Cluster(0, hc.nodes(rng, 4000, (1, 2, 4, 8), MEMS))
    hist = hc.history(rng, cl.nodes, shapes, 6000, 400)
    c_off, units, uids, mut_at, recs = hist
    e = cl.handle()
    e.schedule_batch_mut(c_off, units, mut_at, recs, uids, mode=ROUNDS)
    ref_count, ref_failed, ref_sum = e.headroom(shapes)
    with ShardGroup(cl, world) as g:
        g.each(lambda r, h: h.schedule_batch_mut(c_off, units, mut_at, recs, uids, mode=ROUNDS))
        res = g.each(lambda r, h: h.headroom(shapes, g.ranges[r][0], g.ranges[r][1] - g.ranges[r][0]))
        assert np.array_equal(sum(s for _, _, s in res), ref_sum)
        assert np.array_equal(np.concatenate([c for c, _, _ in res], 1), ref_count)
        assert np.array_equal(np.concatenate([f for _, f, _ in res], 1), ref_failed)

        def outside(r, h):
            lo, hi = g.ranges[r]
            for node0, n in ((0, cl.n_nodes), (hi - 1, 2) if hi < cl.n_nodes else (lo - 1, 2)):
                with pytest.raises(cap.EgsError) as ex:
                    h.headroom(shapes[:1], node0, n)
                assert ex.value.status == cap.EGS_ERR_BAD_ARG
            return True
        assert all(g.each(outside))


# ------------------------------------------------------------------------------------------------ 6. refusals
def test_refusals():
    cap = egs().capi
    N = 1000                                                    # not a multiple of 64
    _, e, uids = with_history(90, N, small_mix(), ROUNDS)
    L, p = e.L, cap._p
    shapes = small_mix()
    c_off = np.array([0, 1, 2], np.int32)
    units = cap.units_array([(25, 4096, 0), (0, 0, 1)])
    cnt = np.zeros((2, N), np.int32); fl = np.zeros((2, N), np.int32); sm = np.zeros((2, 4), np.int64)
    words = cap.node_set_words(N)
    beyond = np.zeros(words, np.uint64); beyond[-1] = np.uint64(1 << 63)
    before = _state(e, shapes, uids[:50])

    def call(n_shapes=2, off=c_off, u=units, node0=0, n=N, bm=None, limit=100, outs=(cnt, fl, sm)):
        return L.egs_headroom(e.h, n_shapes, p(off), p(u), node0, n, p(bm), limit, *[p(x) for x in outs])
    assert call() == cap.EGS_OK
    cases = dict(no_shape=dict(n_shapes=0), empty_shape=dict(off=np.array([0, 0, 1], np.int32)),
                 too_many=dict(off=np.array([0, 5, 6], np.int32), u=cap.units_array([(10, 1, 0)] * 6)),
                 below=dict(node0=-1, n=10), past=dict(node0=N - 5, n=10), negative_n=dict(n=-1),
                 set_bit=dict(bm=beyond), limit_0=dict(limit=0), limit_big=dict(limit=cap.EGS_HEADROOM_MAX_LIMIT + 1),
                 no_output=dict(outs=(None, None, None)))
    for what, kw in cases.items():
        assert call(**kw) == cap.EGS_ERR_BAD_ARG, what
        assert L.egs_last_error(e.h), what
    _same(before, _state(e, shapes, uids[:50]), "a refused call changed the state")
    assert call(limit=cap.EGS_HEADROOM_MAX_LIMIT) == cap.EGS_OK

    s = Cluster(0, hc.nodes(np.random.default_rng(91), 200), c_max=8).handle()
    with pytest.raises(cap.EgsError) as ex:
        s.headroom([[SENT] * 5])                                # 2^15 leaves: the leaf-split Trade
    assert ex.value.status == cap.EGS_ERR_BAD_ARG and b"leaf-split" in s.L.egs_last_error(s.h)
    c, _, _ = s.headroom([[SENT] * 4], limit=3)                 # 2^12 leaves: the one-thread Trade
    assert (c == 3).all()
