"""The rounds ALGORITHM (tests/rounds_model.py, a Python model of csrc/egs_rounds.cuh) is exact: on random
clusters and pod streams -- mixed shapes, sentinel and whole-GPU units, several batches on one state, tiny
list depth / tracked table / shape set so that every early-termination path fires, 1..3 shards -- it
reproduces the reference driver rule (oracle) output for output, digests included."""
import numpy as np
import pytest

import egs_oracle as po
from rounds_model import RoundsModel


def _cluster(rng, n_nodes):
    nodes = []
    for _ in range(n_nodes):
        g = int(rng.choice([1, 2, 4, 8]))
        m = int(rng.choice([16, 40, 80]))
        rows = None
        if rng.integers(0, 2):
            rows = ([int(rng.choice([100, 100, 60, 30, 0])) for _ in range(g)], [int(rng.integers(0, m + 1)) for _ in range(g)])
        nodes.append((100 * g, m * g, rows))
    return nodes


def _shapes(rng, n, mono):
    out = []
    for _ in range(n):
        units = []
        for _ in range(int(rng.integers(1, 4))):
            k = rng.integers(0, 10)
            if k == 0 and not mono:
                units.append((-1, -1, 0))
            elif k == 1:
                units.append((0, 0, int(rng.integers(1, 3))))
            else:
                units.append((int(rng.choice([0, 5, 10, 25, 50])), int(rng.integers(1, 12)), 0))
        out.append(tuple(units))
    return out


@pytest.mark.parametrize("seed", range(24))
def test_model_equals_oracle(seed):
    rng = np.random.default_rng(seed)
    policy = seed % 2
    mono = seed % 3 == 0
    K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
    nodes = _cluster(rng, int(rng.integers(3, 40)))
    shapes = _shapes(rng, int(rng.integers(1, 7)), mono)
    o = po.Scheduler(policy)
    m = RoundsModel(policy, K=K, T=T, RS=RS, shards=D)
    for core, mem, rows in nodes:
        a, b = o.add_node(core, mem), m.add_node(core, mem)
        assert a == b
        if rows:
            o.set_rows(a, *rows); m.set_rows(a, *rows)
    uid = 0
    for batch in range(3):                                        # state (rows, option caches) carries over
        pods = [shapes[int(i)] for i in rng.integers(0, len(shapes), int(rng.integers(20, 160)))]
        got = m.schedule_batch(pods)
        for p, (s, g) in enumerate(zip(pods, got)):
            r = o.schedule_one(list(s), uid)
            uid += 1
            want = dict(node=r["node"], status=r["status"], alloc=r["alloc"], fit_count=r["fit_count"],
                        fit_digest=r["fit_digest"], score_digest=r["score_digest"])
            assert g == want, (seed, batch, p, K, T, RS, D)
        for n in range(len(nodes)):
            assert m.rows(n) == o.rows(n)
        # option caches agree too: cached (CACHED) <=> present in the oracle's map, with the same option
        for s in set(pods):
            for n in range(len(nodes)):
                e = m.tables[s][n]
                opt = o.nodes[n].allocated.get(tuple(s)) if o.nodes[n] is not None else None
                assert (e.st == 1) == (opt is not None), (seed, batch, s, n, e.st)
                if opt is not None:
                    assert (e.score, e.alloc) == (opt.score, opt.allocated)
    assert m.stats["rounds"] >= 3


def test_early_termination_paths_are_exercised():
    tot = dict(rounds=0, dry=0, dry_harmless=0, full=0, shape=0, fast=0)
    for seed in range(24):
        rng = np.random.default_rng(seed)
        K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
        nodes = _cluster(rng, int(rng.integers(3, 40)))
        shapes = _shapes(rng, int(rng.integers(1, 7)), seed % 3 == 0)
        m = RoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D)
        for core, mem, rows in nodes:
            a = m.add_node(core, mem)
            if rows:
                m.set_rows(a, *rows)
        m.schedule_batch([shapes[int(i)] for i in rng.integers(0, len(shapes), 150)])
        for k in tot:
            tot[k] += m.stats[k]
    assert tot["dry"] > 0 and tot["dry_harmless"] > 0 and tot["full"] > 0 and tot["shape"] > 0 and tot["fast"] > 0, tot


def _fast_regime(seed):
    rng = np.random.default_rng(5000 + seed)
    K, T, D = int(rng.choice([1, 2, 4])), int(rng.choice([2, 3, 4, 6])), int(rng.choice([1, 2, 3]))
    nodes = _cluster(rng, int(rng.integers(6, 30)))
    shapes = [((int(rng.choice([5, 10, 25, 50])), int(rng.integers(1, 12)), 0),) for _ in range(int(rng.integers(1, 5)))]
    pods = [shapes[int(i)] for i in rng.integers(0, len(shapes), 200)]
    return K, T, D, nodes, pods


@pytest.mark.parametrize("seed", range(16))
def test_fast_pods_full_table_and_dry_lists_stay_exact(seed):
    """Monotone rounds of single-container shapes (the benchmark regime): fast pods go on resolving on a FULL tracked
    table as long as tracked options win, and an exhausted truncated list ends the round only when what it hides could
    beat the winner -- output for output the oracle's."""
    policy = seed % 2
    K, T, D, nodes, pods = _fast_regime(seed)
    o = po.Scheduler(policy)
    m = RoundsModel(policy, K=K, T=T, RS=8, shards=D)
    for core, mem, rows in nodes:
        a = o.add_node(core, mem); m.add_node(core, mem)
        if rows:
            o.set_rows(a, *rows); m.set_rows(a, *rows)
    got = m.schedule_batch(pods)
    for p, (s, g) in enumerate(zip(pods, got)):
        r = o.schedule_one(list(s), p)
        want = dict(node=r["node"], status=r["status"], alloc=r["alloc"], fit_count=r["fit_count"],
                    fit_digest=r["fit_digest"], score_digest=r["score_digest"])
        assert g == want, (seed, p, K, T, D)
    for n in range(len(nodes)):
        assert m.rows(n) == o.rows(n)
    assert m.stats["fast"] > 0


def test_fast_regime_paths_are_exercised():
    tot = dict(dry=0, dry_harmless=0, full=0, fast=0)
    for seed in range(16):
        K, T, D, nodes, pods = _fast_regime(seed)
        m = RoundsModel(seed % 2, K=K, T=T, RS=8, shards=D)
        for core, mem, rows in nodes:
            a = m.add_node(core, mem)
            if rows:
                m.set_rows(a, *rows)
        m.schedule_batch(pods)
        for k in tot:
            tot[k] += m.stats[k]
    assert all(v > 0 for v in tot.values()), tot


# ------------------------------------------------------------------------------------------------ GPUs above their totals
# A GPU can hold more than its totals: a container without a GPU request (the (-1, -1) sentinel) ADDS 1 to the GPU it
# lands on (gpu.go:36-37), ForgetPod gives back what a failed AddPod never took (node.go:149-150, gpu.go:177-191), and a
# loaded row may be anything up to the int32 guard.  Such a GPU is not free for a whole-GPU container (gpu.go:193-202)
# until a fractional bind brings it down to exactly its totals -- so a round whose requests are all >= 0 can still turn
# an option that did not fit into one that fits.
SIDECAR, WHOLE1, FRAC11 = ((-1, -1, 0),), ((0, 0, 1),), ((1, 1, 0),)
MINIMAL = [[SIDECAR], [WHOLE1, FRAC11, WHOLE1]]   # one node, one GPU of 16 MiB: (101, 17) after batch 1


def replay(m, o, batches, tag, uid=0):
    """Each batch through the model and the oracle: outputs, rows and option caches equal after every batch, and no
    option the model memoises as UNFIT fits the oracle's rows.  Returns the number of whole-GPU pods the oracle bound
    on a node that had a GPU above its totals when the batch began."""
    n_regime = 0
    for b, pods in enumerate(batches):
        over = [o.nodes[n] is not None and any(g.core_avail > g.core_total or g.mem_avail > g.mem_total for g in o.nodes[n].gpus)
                for n in range(len(m.nodes))]
        got = m.schedule_batch(pods)
        for p, (s, g) in enumerate(zip(pods, got)):
            r = o.schedule_one(list(s), uid)
            uid += 1
            want = dict(node=r["node"], status=r["status"], alloc=r["alloc"], fit_count=r["fit_count"],
                        fit_digest=r["fit_digest"], score_digest=r["score_digest"])
            assert g == want, tag + (b, p)
            n_regime += r["status"] == po.EGS_OK and over[r["node"]] and any(u[2] > 0 for u in s)
        for n in range(len(m.nodes)):
            assert m.rows(n) == o.rows(n), tag + (b, n)
        for s in set(pods):
            for n in range(len(m.nodes)):
                e = m.tables[s][n]
                opt = o.nodes[n].allocated.get(tuple(s)) if o.nodes[n] is not None else None
                assert (e.st == 1) == (opt is not None), tag + (b, s, n, e.st)
                if opt is not None:
                    assert (e.score, e.alloc) == (opt.score, opt.allocated), tag + (b, s, n)
                if e.st == 2:
                    assert po.trade(o.nodes[n].gpus, po.RATERS[m.policy], list(s)) is None, tag + (b, s, n, "unfit fits")
    return n_regime


@pytest.mark.parametrize("policy", [0, 1])
def test_whole_gpu_fits_again_after_bind_above_totals(policy):
    """Batch 1 binds a sidecar on the only GPU: (101, 17) of (100, 16).  Batch 2, one round of requests >= 0: a
    whole-GPU pod finds no free GPU; a (1, 1) pod brings the GPU to (100, 16); the next whole-GPU pod takes it.  The
    first pod's "does not fit" must not outlive the second pod's bind."""
    o, m = po.Scheduler(policy), RoundsModel(policy)
    assert o.add_node(100, 16) == m.add_node(100, 16) == 0
    assert replay(m, o, MINIMAL, ("minimal", policy)) == 1
    assert o.rows(0) == [(0, 0)]


OVER = (0, 0, 1, 1, 1, 2, 3)   # how far a GPU starts above its totals, per row


def over_totals_cluster(rng, n_nodes):
    """Nodes of 1, 2 or 4 GPUs whose every GPU is at or just above its totals: core 100..103, memory mt..mt+3, most
    of them 1 above."""
    nodes = []
    for _ in range(n_nodes):
        g, mt = int(rng.choice([1, 2, 4])), int(rng.choice([8, 16]))
        rows = ([100 + int(rng.choice(OVER)) for _ in range(g)], [mt + int(rng.choice(OVER)) for _ in range(g)])
        nodes.append((100 * g, mt * g, rows))
    return nodes


def over_totals_shapes(rng, n):
    """n distinct shapes, every request >= 0: whole-GPU containers of count 1 or 2 (alone or with one fractional
    container), and 1-3 fractional containers of 0-3 core and 0-3 MiB, mostly 0-1 -- small enough to bring a GPU
    just above its totals back to them.  The first two are WHOLE1 and FRAC11, which undoes the most common excess."""
    def frac():
        while True:
            u = (int(rng.choice(OVER)), int(rng.choice(OVER)), 0)
            if u[0] or u[1]:
                return u
    out = [WHOLE1, FRAC11]
    while len(out) < n:
        if rng.integers(0, 2):
            sh = ((0, 0, int(rng.integers(1, 3))),) + ((frac(),) if rng.integers(0, 3) == 0 else ())
        else:
            sh = tuple(frac() for _ in range(int(rng.integers(1, 4))))
        if sh not in out:
            out.append(sh)
    return out


def over_totals_scenario(seed):
    """(policy, K, T, RS, D, nodes, batches): three batches on one state at the tiny list depth / tracked table /
    shape set of test_model_equals_oracle."""
    rng = np.random.default_rng(9000 + seed)
    K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
    nodes = over_totals_cluster(rng, int(rng.integers(3, 24)))
    shapes = over_totals_shapes(rng, int(rng.integers(2, 7)))
    batches = [[shapes[int(i)] for i in rng.integers(0, len(shapes), int(rng.integers(20, 120)))] for _ in range(3)]
    return seed % 2, K, T, RS, D, nodes, batches


def load_over_totals(m, o, nodes):
    for core, mem, rows in nodes:
        a, b = o.add_node(core, mem), m.add_node(core, mem)
        assert a == b
        o.set_rows(a, *rows); m.set_rows(a, *rows)


def _over_totals_run(seed):
    policy, K, T, RS, D, nodes, batches = over_totals_scenario(seed)
    o, m = po.Scheduler(policy), RoundsModel(policy, K=K, T=T, RS=RS, shards=D)
    load_over_totals(m, o, nodes)
    return replay(m, o, batches, (seed, K, T, RS, D))


@pytest.mark.parametrize("seed", range(32))
def test_over_totals_model_equals_oracle(seed):
    _over_totals_run(seed)


def test_over_totals_scenarios_reach_the_regime():
    """Most scenarios bind a whole-GPU pod on a node that began its batch with a GPU above its totals."""
    hits = [_over_totals_run(seed) for seed in range(32)]
    assert sum(h > 0 for h in hits) >= 24, hits
