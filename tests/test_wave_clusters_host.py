"""CPU self-test of tests/wave_clusters.py: the wave arithmetic mirrors select_grid, every planted case has the
property it is built on, and on a small part (n_sm = 2, so the oracle is cheap) the oracle's answers on each planted
cluster differ from its answers on the cluster transformed by that case's mutant.  So each GPU test of
tests/test_gpu_large_clusters.py fails on the defect its case names."""
import numpy as np
import pytest

from oracle_harness import FIELDS
from wave_clusters import CASES, CHUNK, SEL_WARPS, chunk_geometry, chunks_per_warp, sizes, wave

N_SMS = [2, 114, 132]


def _select_grid(n_nodes, n_sm):
    """select_grid of egs_rounds_impl.cuh restated: ceil(chunks / SEL_WARPS) CTAs, at most 2 per SM, at least 1."""
    chunks = -(-n_nodes // 128)
    return max(1, min(-(-chunks // 4), 2 * n_sm))


@pytest.mark.parametrize("n_sm", N_SMS)
def test_chunks_per_warp_mirrors_select_grid(n_sm):
    W = wave(n_sm)
    assert W == 1024 * n_sm
    for n, want in [(W - 1, 1), (W, 1), (W + 1, 2), (2 * W + 127, 3), (1, 1), (129, 1)]:
        nwarps = 4 * _select_grid(n, n_sm)
        chunks = -(-n // 128)
        direct = max(len(range(w, chunks, nwarps)) for w in range(nwarps))   # chunk loop of k_select, per warp
        assert chunks_per_warp(n, n_sm) == direct == want, (n_sm, n)


def _fits(cl, shape):
    o = cl.oracle()
    return o.filter(None, list(shape)).astype(bool)


@pytest.mark.parametrize("n_sm", N_SMS)
def test_planted_properties(n_sm):
    W = wave(n_sm)
    nwarps = 8 * n_sm
    for N in sizes(n_sm):
        assert chunks_per_warp(N, n_sm) >= 2
        warp, pas, _ = chunk_geometry(N, n_sm)
        for policy in (0, 1):
            a = CASES["A"](N, n_sm, policy)
            fit_any = np.zeros(N, bool)
            w = a.cluster.workload
            # below the wave every GPU is at core 0: no fractional or whole-GPU unit fits there
            assert (w.core[:W] == 0).all()
            if n_sm == 2:
                for sh in a.shapes:
                    fit_any |= _fits(a.cluster, sh)
                assert not fit_any[:W].any()
                assert fit_any[W]
            if N == W + 1:
                assert (w.core[W] > 0).any()
            else:
                fit = (w.core > 0).any(1)
                assert len(np.unique(warp[fit])) > nwarps // 2
                assert len(np.unique(np.arange(N)[fit] % 32)) == 32
                assert fit[2 * W:].any() and (pas[fit] == 2).any()          # the partial third chunk
            b = CASES["B"](N, n_sm, policy)
            w = b.cluster.workload
            assert (w.core[:W] == 100).all() and (w.mem[:W] == 8).all()
            assert (w.core[W:, 0] == 100).all() and (w.mem[W:, 0] == 64).all()
            c = CASES["C"](N, n_sm, policy)
            w = c.cluster.workload
            top = (w.core[:, 0] == 100) & (w.core[:, 1:] == 0).all(1) & (w.mem[:, 0] == 64)
            dead = (w.core == 0).all(1)
            assert top.sum() > 128
            assert dead[(pas == 0) & (warp % 2 == 1)].all() and not dead[pas >= 1].any()
            assert top[pas >= 1].any() and top[(pas == 0) & (warp % 2 == 0)].any()
            for name in ("D40", "D110"):
                d = CASES[name](N, n_sm, policy)
                assert len(d.shapes) == int(name[1:])
                assert len(set(d.shapes)) == len(d.shapes)
                assert len(d.c_off) - 1 >= len(d.shapes)


def _first_difference(ref, got):
    P = len(ref["node"])
    bad = [int(np.nonzero(ref[f] != got[f])[0][0]) for f in FIELDS if (ref[f] != got[f]).any()]
    return min(bad) if bad else P


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("case", list(CASES))
def test_mutant_changes_the_answer(case, policy):
    """The oracle on the planted cluster against the oracle on the mutant's cluster: they must differ within the
    first four pods, and for C the winner itself must differ (C's mutant keeps the fit counts of the defect)."""
    n_sm = 2
    for N in sizes(n_sm):
        p = CASES[case](N, n_sm, policy)
        ref = p.cluster.oracle().schedule_batch(p.c_off, p.units.astype(np.int64))
        mut = p.mutant(p.cluster).oracle().schedule_batch(p.c_off, p.units.astype(np.int64))
        if case == "C":
            assert (ref["node"][:4] != mut["node"][:4]).any(), (N, ref["node"][:4], mut["node"][:4])
        else:
            assert _first_difference(ref, mut) < 4, (N, case)
        assert (ref["status"] == 0).any()


def test_generators_prefix_stable():
    """A planted cluster is a prefix of the same case at a larger size, and the batch does not depend on the size."""
    n_sm = 2
    small, large = sizes(n_sm)
    for name, f in CASES.items():
        a, b = f(small, n_sm, 0), f(large, n_sm, 0)
        assert np.array_equal(a.cluster.workload.core, b.cluster.workload.core[:small]), name
        assert np.array_equal(a.cluster.workload.mem, b.cluster.workload.mem[:small]), name
        assert np.array_equal(a.c_off, b.c_off) and np.array_equal(a.units, b.units), name
        shorter = f(small, n_sm, 0, n_pods=50)
        assert np.array_equal(shorter.c_off, a.c_off[:51]) and np.array_equal(shorter.units, a.units[:a.c_off[50]])
    assert CHUNK * SEL_WARPS * 2 == wave(1)
