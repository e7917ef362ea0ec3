"""The mutation stream (SURVEY 8f row 3; controller.go:154-185,301-331): AddPod / ForgetPod records applied in bulk
with one launch, start-up replay of 10^5 assumed pods, and a batch with 10 % mutations woven between its pods -- all
checked against the oracle doing the same thing call by call."""
import numpy as np
import pytest

from oracle_harness import FIELDS, Cluster, compare_outputs, compare_rows, egs

pytestmark = pytest.mark.gpu


def _pair(w):
    cl = Cluster.of_workload(w)
    return cl.handle(), cl.oracle()


def test_bulk_replay_of_assumed_pods_single_launch():
    """scheduler.go:86-106 / node.go:52-54: a restarted scheduler replays every assumed pod onto its node.  10^5
    records (some not fitting any more, some duplicated uids, a few ForgetPods in between) in ONE launch."""
    eg = egs(); cap = eg.capi
    w = eg.workloads.config(4, n_nodes=10_000, n_pods=1)
    e, o = _pair(w)
    rng = np.random.default_rng(7)
    recs, live = [], []
    for i in range(100_000):
        k = rng.integers(0, 20)
        if k == 0 and live:                                       # ForgetPod of an earlier record
            uid, node, req, alloc = live.pop(int(rng.integers(0, len(live))))
            recs.append((cap.EGS_MUT_FORGET, node, req, alloc, uid))
            o.forget_pod(node, req, alloc, uid)
            continue
        node = int(rng.integers(0, w.n_nodes))
        if k == 1:
            req = [(0, 0, int(rng.integers(1, 3)))]
            alloc = [[int(x) for x in sorted(rng.choice(8, size=req[0][2], replace=False))]]
        elif k == 2:
            req = [(-1, -1, 0), (int(rng.choice([10, 25])), 2048, 0)]
            alloc = [[int(rng.integers(0, 8))], [int(rng.integers(0, 8))]]
        else:
            req = [(int(rng.choice([0, 10, 25, 50])), int(rng.choice([4096, 8192, 16384, 40960])), 0)]
            alloc = [[int(rng.integers(0, 8))]]
        uid = 10_000_000 + (i if k != 3 else max(0, i - 5))       # k == 3: a uid seen before -> no-op
        recs.append((cap.EGS_MUT_ADD, node, req, alloc, uid))
        o.add_pod(node, req, alloc, uid)
        live.append((uid, node, req, alloc))
    before = e.profile_get(0)
    assert e.mutations_apply(recs) == 0
    compare_rows(e, o, range(w.n_nodes))
    for uid, _, _, _ in live[:200]:
        assert e.pod_known(uid) == o.known_pod(uid)
    assert before == e.profile_get(0)


def test_batch_with_ten_percent_mutations_interleaved():
    """50 000 pods with ~5 000 AddPod / ForgetPod records woven in at fixed pod positions: the oracle runs segment by
    segment with the single-pod verbs in between (the order the reference's lock gives), the GPU takes the whole
    stream in one call."""
    eg = egs(); cap = eg.capi
    w = eg.workloads.config(4, n_nodes=2_000, n_pods=50_000)
    e, o = _pair(w)
    rng = np.random.default_rng(11)
    P = w.n_pods
    cuts = sorted(set(int(x) for x in rng.integers(1, P, 5_000)))
    uids = np.arange(1, P + 1, dtype=np.uint64)
    ref = {f: [] for f in FIELDS}
    recs, mut_at = [], []
    bound = []                                                    # (uid, node, req, alloc) of pods the oracle bound
    ext = 0
    prev = 0
    for cut in cuts + [P]:
        seg = eg.workloads.window(w, prev, cut - prev)
        r = o.schedule_batch(seg.c_off, seg.units64(), uids=uids[prev:cut])
        for f in FIELDS:
            ref[f].append(r[f])
        for i in range(seg.n_pods):
            if r["status"][i] == 0:
                req = [tuple(int(x) for x in seg.units[k]) for k in range(int(seg.c_off[i]), int(seg.c_off[i + 1]))]
                alloc = cap.masks_to_lists(r["alloc_mask"][i], len(req))
                bound.append((int(uids[prev + i]), int(r["node"][i]), req, alloc))
        prev = cut
        if cut == P:
            break
        if rng.integers(0, 3) and bound:                          # ForgetPod of a pod scheduled earlier in this very batch
            uid, node, req, alloc = bound.pop(int(rng.integers(0, len(bound))))
            recs.append((cap.EGS_MUT_FORGET, node, req, alloc, uid)); mut_at.append(cut)
            o.forget_pod(node, req, alloc, uid)
        else:                                                     # AddPod of a pod another scheduler bound
            ext += 1
            node = int(rng.integers(0, w.n_nodes))
            req = [(int(rng.choice([10, 25, 50])), int(rng.choice([4096, 16384])), 0)]
            alloc = [[int(rng.integers(0, 8))]]
            recs.append((cap.EGS_MUT_ADD, node, req, alloc, 5_000_000 + ext)); mut_at.append(cut)
            o.add_pod(node, req, alloc, 5_000_000 + ext)
    got = e.schedule_batch_mut(w.c_off, w.units, mut_at, recs, uids=uids)
    compare_outputs({f: np.concatenate(ref[f]) for f in FIELDS}, got, "batch with mutations")
    compare_rows(e, o, range(w.n_nodes))
    assert len(recs) > 4_000
