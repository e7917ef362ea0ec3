"""Pre-install (k_resolve_mw's prologue tracks the round's likely winners before the first pod) is exact: the rounds
model with pre-install (tests/rounds_model_preinstall.py) reproduces the reference driver rule output for output on
the scenarios of tests/test_rounds_model.py, with nothing, one rank or whole lists pre-installed and with the tracked
table up to one slot short of full before the first pod -- while every early stop (table full, list dry, shape
outside the set) still fires with pre-installed slots present."""
import numpy as np
import pytest

import egs_oracle as po
from rounds_model import RoundsModel
from rounds_model_preinstall import PreinstallRoundsModel
from test_rounds_model import MINIMAL, _cluster, _fast_regime, _shapes, load_over_totals, over_totals_scenario, replay

PRE_H = (0, 1, 64)                                                # off, the top of every list, every list entry


def _cap(T, which):
    return T - 1 if which == "full" else max(1, T // 2)


def _check(m, o, pods, uid0, tag):
    got = m.schedule_batch(pods)
    for p, (s, g) in enumerate(zip(pods, got)):
        r = o.schedule_one(list(s), uid0 + p)
        want = dict(node=r["node"], status=r["status"], alloc=r["alloc"], fit_count=r["fit_count"],
                    fit_digest=r["fit_digest"], score_digest=r["score_digest"])
        assert g == want, tag + (p,)
    return uid0 + len(pods)


@pytest.mark.parametrize("cap", ["full", "half"])
@pytest.mark.parametrize("pre_h", PRE_H)
@pytest.mark.parametrize("seed", range(24))
def test_preinstall_model_equals_oracle(seed, pre_h, cap):
    rng = np.random.default_rng(seed)                             # the scenarios of test_model_equals_oracle
    policy = seed % 2
    mono = seed % 3 == 0
    K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
    nodes = _cluster(rng, int(rng.integers(3, 40)))
    shapes = _shapes(rng, int(rng.integers(1, 7)), mono)
    o = po.Scheduler(policy)
    m = PreinstallRoundsModel(policy, K=K, T=T, RS=RS, shards=D, pre_h=pre_h, pre_cap=_cap(T, cap))
    for core, mem, rows in nodes:
        a, b = o.add_node(core, mem), m.add_node(core, mem)
        assert a == b
        if rows:
            o.set_rows(a, *rows); m.set_rows(a, *rows)
    uid = 0
    for batch in range(3):
        pods = [shapes[int(i)] for i in rng.integers(0, len(shapes), int(rng.integers(20, 160)))]
        uid = _check(m, o, pods, uid, (seed, pre_h, cap, batch, K, T, RS, D))
        for n in range(len(nodes)):
            assert m.rows(n) == o.rows(n)
        for s in set(pods):                                       # option caches agree too
            for n in range(len(nodes)):
                e = m.tables[s][n]
                opt = o.nodes[n].allocated.get(tuple(s)) if o.nodes[n] is not None else None
                assert (e.st == 1) == (opt is not None), (seed, batch, s, n, e.st)
                if opt is not None:
                    assert (e.score, e.alloc) == (opt.score, opt.allocated)
    assert (m.stats["pre"] > 0) == (pre_h > 0)


@pytest.mark.parametrize("pre_h", PRE_H[1:])
@pytest.mark.parametrize("seed", range(16))
def test_preinstall_fast_regime_equals_oracle(seed, pre_h):
    policy = seed % 2
    K, T, D, nodes, pods = _fast_regime(seed)
    o = po.Scheduler(policy)
    m = PreinstallRoundsModel(policy, K=K, T=T, RS=8, shards=D, pre_h=pre_h)
    for core, mem, rows in nodes:
        a = o.add_node(core, mem); m.add_node(core, mem)
        if rows:
            o.set_rows(a, *rows); m.set_rows(a, *rows)
    _check(m, o, pods, 0, (seed, pre_h, K, T, D))
    for n in range(len(nodes)):
        assert m.rows(n) == o.rows(n)


@pytest.mark.parametrize("pre_h", PRE_H[1:])
def test_stops_fire_with_preinstalled_slots(pre_h):
    tot = dict(rounds=0, dry=0, dry_harmless=0, full=0, shape=0, fast=0, pre=0)
    for seed in range(24):
        rng = np.random.default_rng(seed)
        K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
        nodes = _cluster(rng, int(rng.integers(3, 40)))
        shapes = _shapes(rng, int(rng.integers(1, 7)), seed % 3 == 0)
        m = PreinstallRoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D, pre_h=pre_h)
        for core, mem, rows in nodes:
            a = m.add_node(core, mem)
            if rows:
                m.set_rows(a, *rows)
        m.schedule_batch([shapes[int(i)] for i in rng.integers(0, len(shapes), 150)])
        for k in tot:
            tot[k] += m.stats[k]
    assert all(v > 0 for v in tot.values()), tot


@pytest.mark.parametrize("pre_h", PRE_H)
@pytest.mark.parametrize("policy", [0, 1])
def test_preinstall_whole_gpu_fits_again_after_bind_above_totals(policy, pre_h):
    """test_rounds_model's minimal case with the node pre-installed: a GPU at (101, 17) of (100, 16) is not free for
    the first whole-GPU pod, is after a (1, 1) bind, and the second whole-GPU pod takes it."""
    o, m = po.Scheduler(policy), PreinstallRoundsModel(policy, pre_h=pre_h)
    assert o.add_node(100, 16) == m.add_node(100, 16) == 0
    assert replay(m, o, MINIMAL, ("minimal", policy, pre_h)) == 1
    assert o.rows(0) == [(0, 0)]


@pytest.mark.parametrize("cap", ["full", "half"])
@pytest.mark.parametrize("pre_h", PRE_H)
@pytest.mark.parametrize("seed", range(16))
def test_preinstall_over_totals_equals_oracle(seed, pre_h, cap):
    """GPUs at or just above their totals, whole-GPU and small fractional shapes only (every round's requests >= 0),
    three batches on one state: outputs, rows, caches and UNFIT memos equal the oracle's."""
    policy, K, T, RS, D, nodes, batches = over_totals_scenario(seed)
    o = po.Scheduler(policy)
    m = PreinstallRoundsModel(policy, K=K, T=T, RS=RS, shards=D, pre_h=pre_h, pre_cap=_cap(T, cap))
    load_over_totals(m, o, nodes)
    replay(m, o, batches, (seed, pre_h, cap, K, T, RS, D))
    assert (m.stats["pre"] > 0) == (pre_h > 0)


@pytest.mark.parametrize("seed", range(24))
def test_preinstall_off_is_the_rounds_model(seed):
    """pre_h = 0: the same outputs, rounds and stops as tests/rounds_model.py, so the two models cannot drift apart."""
    rng = np.random.default_rng(seed)
    K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
    nodes = _cluster(rng, int(rng.integers(3, 40)))
    shapes = _shapes(rng, int(rng.integers(1, 7)), seed % 3 == 0)
    a, b = RoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D), PreinstallRoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D)
    for core, mem, rows in nodes:
        for m in (a, b):
            n = m.add_node(core, mem)
            if rows:
                m.set_rows(n, *rows)
    for _ in range(3):
        pods = [shapes[int(i)] for i in rng.integers(0, len(shapes), int(rng.integers(20, 160)))]
        assert a.schedule_batch(pods) == b.schedule_batch(pods)
    assert a.stats == {k: v for k, v in b.stats.items() if k != "pre"} and b.stats["pre"] == 0
