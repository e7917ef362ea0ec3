"""One handle under the extender's interleaved call stream (tests/call_stream.py), every answer against the C oracle:
Filter / Score / Bind, AddPod / ForgetPod / replay and mutation records, node reloads, batches through all five entry
points, checkpoint what-ifs, headroom and eviction what-ifs, all on the same per-handle state -- option tables and their
"known not to fit" memos, cold slots, pending batches' uid bookkeeping, shape interning past 256 shapes, and the scratch
buffers every entry point shares.

  1. a serial stream on every geometry and policy, with rows, option tables and uid bookkeeping checked every 500
     steps and at the end;
  2. the same stream with each call issued from a random thread of eight (egs.h: any OS thread);
  3. concurrent callers: threads on one handle at once, each on its own interleaved node partition and uid range,
     each answer equal to the oracle running the sub-streams one after the other;
  4. a cluster one node past a k_select wave, so the hand-offs also run where the select, merge and pass kernels
     change shape.
Each stream prints what it reached: step kinds, statuses, shapes interned, the widest batch."""
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import call_stream as cs
import oracle_c as oc
import wave_clusters as wc
from oracle_harness import compare_caches, compare_rows, egs

pytestmark = pytest.mark.gpu

N_SERIAL = 1341                 # a multiple of neither 64 nor 128: six 256-thread blocks, a partial set word
STEPS = 5000
CHECK_EVERY = 500


# ------------------------------------------------------------------------------------------------ the library side
def handle(m):
    """The stream's initial cluster on a new handle; runs of nodes of one size load in bulk."""
    g = cs.GEOMETRY[m.geo]
    e = egs().Egs(m.policy, m.N, g["g_max"], c_max=g["c_max"])
    nodes, n = m.nodes0, 0
    while n < m.N:
        gc, mt = nodes[n][:2]
        q = n
        while q < m.N and nodes[q][:2] == (gc, mt):
            q += 1
        core = np.array([nd[2][0] if nd[2] else [100] * gc for nd in nodes[n:q]], np.int32)
        mem = np.array([nd[2][1] if nd[2] else [mt] * gc for nd in nodes[n:q]], np.int32)
        e.state_load_bulk(n, gc, mt, core, mem)
        n = q
    return e


def replay_pod(e, node, req, alloc, uid):
    cap = egs().capi
    off, idx = cap._alloc_arrays(alloc)
    return e.L.egs_node_replay_pod(e.h, node, len(req), cap._p(cap.units_array(req)), cap._p(off), cap._p(idx), uid)


def device_batch(e, c_off, units, mode):
    import torch
    P = len(c_off) - 1
    d = dict(node=torch.empty(P, dtype=torch.int32, device="cuda"), status=torch.empty(P, dtype=torch.int32, device="cuda"),
             alloc_mask=torch.empty((P, e.n_masks * e.mask_dtype.itemsize), dtype=torch.uint8, device="cuda"),
             fit_count=torch.empty(P, dtype=torch.int32, device="cuda"),
             fit_digest=torch.empty(P, dtype=torch.int64, device="cuda"),
             score_digest=torch.empty(P, dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    e.schedule_batch_device(c_off, units, [t.data_ptr() for t in d.values()], mode=mode)
    out = {k: t.cpu().numpy() for k, t in d.items()}
    out["alloc_mask"] = out["alloc_mask"].view(e.mask_dtype)
    out["fit_digest"], out["score_digest"] = out["fit_digest"].view(np.uint64), out["score_digest"].view(np.uint64)
    return out


def run(e, step, call=lambda f, *a, **k: f(*a, **k)):
    """`step` on library handle `e`, each library call through `call`; the answer in the form Model.apply gives."""
    k = step["kind"]
    req, ids = step.get("req"), step.get("ids")
    if k == "filter":
        return dict(fit=call(e.filter, ids, req))
    if k in ("filter_score", "schedule_one"):
        fit = call(e.filter, ids, req)
        cand = np.arange(e.max_nodes, dtype=np.int32) if ids is None else np.asarray(ids, np.int32)
        fid = cand[fit.astype(bool)]
        if k == "schedule_one" and len(fid) == 0:
            return dict(fit=fit, status=cs.OK, score=np.zeros(0, np.int64), node=-1, bind=cs.NOFIT, alloc=None)
        st, sc = call(e.score, fid, req)
        if k == "filter_score":
            return dict(fit=fit, status=st, score=sc)
        w = int(fid[int(np.argmax(sc))])
        bst, alloc = call(e.bind, w, req, step["uid"])
        return dict(fit=fit, status=st, score=sc, node=w, bind=bst, alloc=alloc)
    if k == "score":
        st, sc = call(e.score, ids, req)
        return dict(status=st, score=sc)
    if k == "bind":
        st, alloc = call(e.bind, step["node"], req, step["uid"])
        return dict(status=st, alloc=alloc)
    if k == "peek":
        return dict(opt=[call(e.peek, n, req) for n in step["nodes"]])
    if k in ("apply", "replay", "cancel"):
        f = dict(apply=e.pod_apply, cancel=e.pod_cancel)[k] if k != "replay" else \
            (lambda *a: replay_pod(e, *a))
        return dict(status=call(f, step["node"], req, step["alloc"], step["uid"]))
    if k == "records":
        return dict(status=call(e.mutations_apply, step["records"]))
    if k == "reload":
        G, mt = step["gpus"], step["mt"]
        return dict(status=call(e.node_set_allocatable, step["node"], 100 * G, mt * G))
    if k == "load":
        return dict(status=call(e.state_load, step["node"], step["core"], step["mem"]))
    if k == "batch":
        c_off, units = cs.c_off_units(step["reqs"])
        units = units.astype(np.int32)
        entry, mode, uids = step["entry"], step["mode"], step["uids"]
        if entry == "plain":
            out = call(e.schedule_batch, c_off, units, uids=uids, mode=mode)
        elif entry == "nodes":
            out = call(e.schedule_batch_nodes, c_off, units, step["sets"], step["pod_set"], uids=uids, mode=mode)
        elif entry == "mut":
            out = call(e.schedule_batch_mut, c_off, units, step["mut_at"], step["records"], uids=uids, mode=mode)
        elif entry == "vec":
            out = call(e.schedule_batch_vec, c_off, units, step["vec_pods"], uids=uids)
        else:
            out = call(device_batch, e, c_off, units, mode)
        return out
    if k == "headroom":
        count, failed, summary = call(e.headroom, step["shapes"], step["node0"], step["n"], node_set=step["set"],
                                      limit=step["limit"])
        return dict(count=count, failed=failed, summary=summary)
    if k == "evict":
        st, sc, masks = call(e.evict_fit, req, step["ids"], step["victims"])
        assert not masks[st != cs.OK].any(), "evict_fit: masks of a node that does not bind"
        return dict(status=st, score=sc, alloc=[cs.lists_of(m, len(req)) if s == cs.OK else None
                                                for s, m in zip(st.tolist(), masks)])
    if k == "known":
        return dict(known=np.array([call(e.pod_known, u) for u in step["uids"]], bool),
                    released=np.array([call(e.pod_released, u) for u in step["uids"]], bool))
    if k in ("save", "rollback", "drop"):
        call(getattr(e, "checkpoint_" + k))
        return dict(status=cs.OK)
    raise ValueError(k)


def check_state(e, m, uids, what, sample=None, seed=0):
    """Rows of every node, the option table of every interned shape (memos included) on `sample` nodes (None: all),
    podMaps and releasedPodMap of every uid."""
    try:
        compare_rows(e, m.o, range(m.N))
        nodes = range(m.N) if sample is None else \
            np.random.default_rng(seed).choice(m.N, min(sample, m.N), replace=False)
        compare_caches(e, m.o, [list(sh) for sh in m.interned], nodes, unfit_check=True)
        for u in uids:
            assert e.pod_known(u) == m.o.known_pod(u), f"pod_known({u})"
            assert e.pod_released(u) == m.o.released_pod(u), f"pod_released({u})"
    except AssertionError as ex:
        raise AssertionError(f"{what}: {ex}") from None


def drive(s, e, steps, call=None, check_every=CHECK_EVERY, sample=512, final_sample=None):
    call = call or (lambda f, *a, **k: f(*a, **k))
    what = f"seed {s.seed} ({s.geo}, policy {s.model.policy})"
    for i in range(steps):
        step, ref = s.next()
        got = run(e, step, call)
        d = cs.diff(ref, got)
        assert d is None, f"{what}, step {i} ({step['kind']}{':' + step['entry'] if 'entry' in step else ''}): {d}"
        if (i + 1) % check_every == 0:
            check_state(e, s.model, s.used_uids[-2000:], f"{what}, after step {i}", sample, seed=i)
    check_state(e, s.model, s.used_uids + [cs.AUTO_UID0 + k for k in range(64)], f"{what}, at the end", final_sample)


def reached(s):
    """What the stream reached, printed, and the coverage every serial stream must have."""
    rep = s.report()
    print(f"\nseed {s.seed} ({s.geo}, policy {s.model.policy}): {rep}")
    kinds = rep["kinds"]
    for k in s.entries + ["save", "rollback"]:
        assert kinds.get(k, 0) > 0, f"step kind {k} never ran"
    want = {cs.OK, cs.NOFIT, cs.TRANSACT, cs.NO_OPTION, cs.PANIC}
    assert want <= set(rep["statuses"]), f"statuses {rep['statuses']}"
    assert rep["max_shapes"] > cs.SHAPE_CACHE and rep["shapes_past_256_under_checkpoint"], rep
    assert rep["widest_batch"] > cs.RSMAX, rep
    mut = {m for m, _ in s.after}
    missing = [(m, x) for m in mut for x in s.entries if (m, x) not in s.after]
    assert not missing, f"entry points never run after a state change: {missing[:10]}"


# ------------------------------------------------------------------------------------------------ 1. serial
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("geo", ["8", "wide", "sidecar"])
def test_serial_stream(geo, policy):
    t0 = time.time()
    s = cs.Stream(11 + 2 * policy + {"8": 0, "wide": 100, "sidecar": 200}[geo], geo, policy, N_SERIAL, STEPS)
    e = handle(s.model)
    drive(s, e, STEPS)
    reached(s)
    e.close()
    print(f"{STEPS} steps in {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ 2. thread hopping
def test_thread_hopping():
    """Every call from a random worker of eight single-thread pools, one call at a time."""
    s = cs.Stream(31, "8", 0, N_SERIAL, 2500)
    e = handle(s.model)
    pools = [ThreadPoolExecutor(1) for _ in range(8)]
    rng = np.random.default_rng(32)
    threads = set()

    def call(f, *a, **k):
        def on_worker():
            threads.add(threading.get_ident())
            return f(*a, **k)
        return pools[int(rng.integers(8))].submit(on_worker).result()
    try:
        drive(s, e, 2500, call)
    finally:
        for p in pools:
            p.shutdown()
    assert len(threads) == 8
    print(f"\nthread hopping: {s.report()}")
    e.close()


# ------------------------------------------------------------------------------------------------ 3. concurrent
@pytest.mark.parametrize("parts", [4, 8])
def test_concurrent_callers(parts):
    """`parts` threads at once on one handle; thread t owns nodes t, t + parts, ... (shared set words and kernel
    blocks) and its own uids.  Each thread's answers equal the oracle running the sub-streams one after the other,
    and so does the final state."""
    steps = 8000 // parts
    base = cs.Stream(41 + parts, "8", 0, N_SERIAL, steps, part=0, parts=parts)
    subs = [base] + [cs.Stream(41 + parts + t, "8", 0, N_SERIAL, steps, part=t, parts=parts, model=base.model)
                     for t in range(1, parts)]
    plans = [[sub.next() for _ in range(steps)] for sub in subs]
    e = handle(base.model)
    start = threading.Barrier(parts)
    errors = [None] * parts

    def worker(t):
        start.wait()
        for i, (step, ref) in enumerate(plans[t]):
            try:
                d = cs.diff(ref, run(e, step))
            except Exception as ex:                 # pragma: no cover
                d = repr(ex)
            if d is not None:
                errors[t] = f"thread {t} (seed {subs[t].seed}), step {i} ({step['kind']}): {d}"
                return
    th = [threading.Thread(target=worker, args=(t,)) for t in range(parts)]
    for x in th:
        x.start()
    for x in th:
        x.join(timeout=900)
    assert not any(x.is_alive() for x in th)
    bad = [x for x in errors if x]
    assert not bad, bad
    uids = [u for sub in subs for u in sub.used_uids]
    check_state(e, base.model, uids, f"{parts} concurrent callers, at the end")
    for sub in subs:
        assert sub.counts["batch:nodes"] > 0 and sub.counts["evict"] > 0 and sub.counts["headroom"] > 0
    print(f"\n{parts} concurrent callers: {[sub.report()['kinds'] for sub in subs[:1]]}")
    e.close()


# ------------------------------------------------------------------------------------------------ 4. past one wave
def test_past_one_select_wave():
    """wave(n_sm) + 1 nodes: a few hundred steps, mostly batches and full-list filters."""
    import torch
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    N = wc.wave(n_sm) + 1
    rng = np.random.default_rng(51)
    nodes = []
    while len(nodes) < N:                            # runs of 512 nodes of one size: bulk loads
        g, mt = int(rng.choice((2, 4, 8))), int(rng.choice(cs.MEMS))
        block = cs.cluster(rng, 512, (g,), (mt,))
        nodes += block[:N - len(nodes)]
    weights = {k: 0 for k in cs.WEIGHTS}
    weights.update(filter=8, batch=14, schedule_one=2, filter_score=0, score=1, apply=2, cancel=2, records=2,
                   reload=1, load=1, bind=1, peek=1, replay=1, headroom=1, evict=1, known=1)
    s = cs.Stream(52, "8", 0, N, 300, nodes=nodes, big_batch=400, weights=weights, pace=False)
    e = handle(s.model)
    drive(s, e, 300, check_every=100, sample=4096, final_sample=8192)
    print(f"\n{N} nodes: {s.report()}")
    e.close()


# ------------------------------------------------------------------------------------------------ regressions
@pytest.mark.parametrize("mode", [cs.RESCAN, cs.ROUNDS])
def test_regression_rows_below_zero_after_sentinel_forget(mode):
    """The stream's first disagreement, minimised: AddPod of a sentinel pod (+1 on a GPU), the node's rows reloaded,
    ForgetPod of that pod (-1: the GPU goes below zero).  Binpack rates with Go's signed minimum, so the single-
    container Trade must count the negative GPU; it took an unsigned minimum, which skipped it."""
    req = [(10, 4, 0)]
    for k in range(3):
        e, o = egs().Egs(0, 3, 8), oc.OracleC(0)
        for n in range(3):
            assert e.node_set_allocatable(n, 200, 32) == 0 and o.add_node(200, 32) == n
        assert e.pod_apply(1, [cs.SENT], [[1]], 7) == 0 and o.add_pod(1, [cs.SENT], [[1]], 7) == 0
        assert e.state_load(1, [50, 0], [16, 0]) == 0
        o.set_rows(1, [50, 0], [16, 0])
        assert e.pod_cancel(1, [cs.SENT], [[1]], 7) == 0 and o.forget_pod(1, [cs.SENT], [[1]], 7) == 0
        assert e.rows(1) == o.rows(1) == [(50, 16), (-1, -1)]
        if k == 0:                                   # the verbs
            assert list(e.filter(None, req)) == list(o.filter(None, req))
            st, sc = e.score(None, req)
            assert st == 0 and list(sc) == o.score(None, req)[1].tolist()
            assert e.bind(1, req, 8) == o.bind(1, req, 8)
        else:                                        # a batch on tables the verbs did (k == 2) or did not prepare
            if k == 2:
                e.filter(None, req); o.filter(None, req)
            c_off, units = cs.c_off_units([req] * 4)
            ref = o.schedule_batch(c_off, units, uids=np.arange(10, 14, dtype=np.uint64))
            got = e.schedule_batch(c_off, units.astype(np.int32), uids=np.arange(10, 14, dtype=np.uint64), mode=mode)
            for f in ref:
                assert np.array_equal(ref[f], got[f]), f
        assert e.rows(1) == o.rows(1)
        e.close()
