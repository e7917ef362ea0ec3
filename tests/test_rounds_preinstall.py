"""Pre-install (k_resolve_mw's prologue tracks the round's likely winners before the first pod) is exact: the rounds
model with pre-install (tests/rounds_model_preinstall.py) reproduces the reference driver rule output for output on
the scenarios of tests/test_rounds_model.py (built by tests/rounds_cases.py), with nothing, one rank or whole lists
pre-installed and with the tracked table up to one slot short of full before the first pod -- while every early stop
(table full, list dry, shape outside the set) still fires with pre-installed slots present."""
import pytest

import egs_oracle as po
from rounds_cases import MINIMAL, check_batch, fast_regime, load_nodes, model_batches, model_scenario, \
    over_totals_scenario, replay
from rounds_model import RoundsModel
from rounds_model_preinstall import PreinstallRoundsModel

PRE_H = (0, 1, 64)                                                # off, the top of every list, every list entry


def _cap(T, which):
    return T - 1 if which == "full" else max(1, T // 2)


@pytest.mark.parametrize("cap", ["full", "half"])
@pytest.mark.parametrize("pre_h", PRE_H)
@pytest.mark.parametrize("seed", range(24))
def test_preinstall_model_equals_oracle(seed, pre_h, cap):
    rng, K, T, RS, D, nodes, shapes = model_scenario(seed)          # the scenarios of test_model_equals_oracle
    o = po.Scheduler(seed % 2)
    m = PreinstallRoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D, pre_h=pre_h, pre_cap=_cap(T, cap))
    load_nodes(nodes, o, m)
    replay(m, o, model_batches(rng, shapes), (seed, pre_h, cap, K, T, RS, D))
    assert (m.stats["pre"] > 0) == (pre_h > 0)


@pytest.mark.parametrize("pre_h", PRE_H[1:])
@pytest.mark.parametrize("seed", range(16))
def test_preinstall_fast_regime_equals_oracle(seed, pre_h):
    policy = seed % 2
    K, T, D, nodes, pods = fast_regime(seed)
    o = po.Scheduler(policy)
    m = PreinstallRoundsModel(policy, K=K, T=T, RS=8, shards=D, pre_h=pre_h)
    load_nodes(nodes, o, m)
    check_batch(m, o, pods, 0, (seed, pre_h, K, T, D))
    for n in range(len(nodes)):
        assert m.rows(n) == o.rows(n)


@pytest.mark.parametrize("pre_h", PRE_H[1:])
def test_stops_fire_with_preinstalled_slots(pre_h):
    tot = dict(rounds=0, dry=0, dry_harmless=0, full=0, shape=0, fast=0, pre=0)
    for seed in range(24):
        rng, K, T, RS, D, nodes, shapes = model_scenario(seed)
        m = PreinstallRoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D, pre_h=pre_h)
        load_nodes(nodes, m)
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
    load_nodes(nodes, o, m)
    replay(m, o, batches, (seed, pre_h, cap, K, T, RS, D))
    assert (m.stats["pre"] > 0) == (pre_h > 0)


@pytest.mark.parametrize("seed", range(24))
def test_preinstall_off_is_the_rounds_model(seed):
    """pre_h = 0: the same outputs, rounds and stops as tests/rounds_model.py, so the two models cannot drift apart."""
    rng, K, T, RS, D, nodes, shapes = model_scenario(seed)
    a, b = RoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D), PreinstallRoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D)
    load_nodes(nodes, a, b)
    for pods in model_batches(rng, shapes):
        assert a.schedule_batch(pods) == b.schedule_batch(pods)
    assert a.stats == {k: v for k, v in b.stats.items() if k != "pre"} and b.stats["pre"] == 0
