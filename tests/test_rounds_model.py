"""The rounds ALGORITHM (tests/rounds_model.py, a Python model of csrc/egs_rounds.cuh) is exact: on random
clusters and pod streams -- mixed shapes, sentinel and whole-GPU units, several batches on one state, tiny
list depth / tracked table / shape set so that every early-termination path fires, 1..3 shards -- it
reproduces the reference driver rule (oracle) output for output, digests included."""
import pytest

import egs_oracle as po
from rounds_cases import MINIMAL, check_batch, fast_regime, load_nodes, model_batches, model_scenario, \
    over_totals_scenario, replay
from rounds_model import RoundsModel


@pytest.mark.parametrize("seed", range(24))
def test_model_equals_oracle(seed):
    """Three batches on one state (rows, option caches carry over): outputs, rows and option caches equal."""
    rng, K, T, RS, D, nodes, shapes = model_scenario(seed)
    o, m = po.Scheduler(seed % 2), RoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D)
    load_nodes(nodes, o, m)
    replay(m, o, model_batches(rng, shapes), (seed, K, T, RS, D))
    assert m.stats["rounds"] >= 3


def test_early_termination_paths_are_exercised():
    tot = dict(rounds=0, dry=0, dry_harmless=0, full=0, shape=0, fast=0)
    for seed in range(24):
        rng, K, T, RS, D, nodes, shapes = model_scenario(seed)
        m = RoundsModel(seed % 2, K=K, T=T, RS=RS, shards=D)
        load_nodes(nodes, m)
        m.schedule_batch([shapes[int(i)] for i in rng.integers(0, len(shapes), 150)])
        for k in tot:
            tot[k] += m.stats[k]
    assert tot["dry"] > 0 and tot["dry_harmless"] > 0 and tot["full"] > 0 and tot["shape"] > 0 and tot["fast"] > 0, tot


@pytest.mark.parametrize("seed", range(16))
def test_fast_pods_full_table_and_dry_lists_stay_exact(seed):
    """Monotone rounds of single-container shapes (the benchmark regime): fast pods go on resolving on a FULL tracked
    table as long as tracked options win, and an exhausted truncated list ends the round only when what it hides could
    beat the winner -- output for output the oracle's."""
    policy = seed % 2
    K, T, D, nodes, pods = fast_regime(seed)
    o, m = po.Scheduler(policy), RoundsModel(policy, K=K, T=T, RS=8, shards=D)
    load_nodes(nodes, o, m)
    check_batch(m, o, pods, 0, (seed, K, T, D))
    for n in range(len(nodes)):
        assert m.rows(n) == o.rows(n)
    assert m.stats["fast"] > 0


def test_fast_regime_paths_are_exercised():
    tot = dict(dry=0, dry_harmless=0, full=0, fast=0)
    for seed in range(16):
        K, T, D, nodes, pods = fast_regime(seed)
        m = RoundsModel(seed % 2, K=K, T=T, RS=8, shards=D)
        load_nodes(nodes, m)
        m.schedule_batch(pods)
        for k in tot:
            tot[k] += m.stats[k]
    assert all(v > 0 for v in tot.values()), tot


# ------------------------------------------------------------------------------------------------ GPUs above their totals
@pytest.mark.parametrize("policy", [0, 1])
def test_whole_gpu_fits_again_after_bind_above_totals(policy):
    """Batch 1 binds a sidecar on the only GPU: (101, 17) of (100, 16).  Batch 2, one round of requests >= 0: a
    whole-GPU pod finds no free GPU; a (1, 1) pod brings the GPU to (100, 16); the next whole-GPU pod takes it.  The
    first pod's "does not fit" must not outlive the second pod's bind."""
    o, m = po.Scheduler(policy), RoundsModel(policy)
    assert o.add_node(100, 16) == m.add_node(100, 16) == 0
    assert replay(m, o, MINIMAL, ("minimal", policy)) == 1
    assert o.rows(0) == [(0, 0)]


def _over_totals_run(seed):
    policy, K, T, RS, D, nodes, batches = over_totals_scenario(seed)
    o, m = po.Scheduler(policy), RoundsModel(policy, K=K, T=T, RS=RS, shards=D)
    load_nodes(nodes, o, m)
    return replay(m, o, batches, (seed, K, T, RS, D))


@pytest.mark.parametrize("seed", range(32))
def test_over_totals_model_equals_oracle(seed):
    _over_totals_run(seed)


def test_over_totals_scenarios_reach_the_regime():
    """Most scenarios bind a whole-GPU pod on a node that began its batch with a GPU above its totals."""
    hits = [_over_totals_run(seed) for seed in range(32)]
    assert sum(h > 0 for h in hits) >= 24, hits
