"""CPU self-test of tests/sidecar_cases.py: every planted node kind has the property it is built on, every mutant
changes the oracle's answer on its kind, and the cluster sizes give every CTA of k_trade_leaves items of several
misses at any occupancy, for 2, 114 and 132 SMs.  So each GPU test of tests/test_gpu_sidecar_scale.py can fail on
the defect its kind names."""
import numpy as np
import pytest

import oracle_c
from sidecar_cases import KINDS, S5, S6, S8, TIES, TILE, chunk_of, items, leaf_grid_max, leaf_of, n_branch, \
    planted_cluster, planted_nodes, s8_count, several_items_per_cta, tile_of, tiles, warp_of

N_SMS = [2, 114, 132]


def _trade(rows, shape, policy):
    o = oracle_c.OracleC(policy)
    n = o.add_node(100 * len(rows), 32 * len(rows))
    o.set_rows(n, [c for c, _ in rows], [m for _, m in rows])
    return o.trade(n, list(shape))


def test_tiles_per_shape():
    assert [n_branch(s) for s in (S5, S6, S8)] == [5, 6, 8]
    assert [tiles(s) for s in (S5, S6, S8)] == [2, 16, 1024]
    assert TILE == 1 << 14


@pytest.mark.parametrize("n_sm", N_SMS)
def test_every_cta_takes_items_of_several_misses(n_sm):
    """A cold Trade over every node of the planted cluster, and S8 over s8_count nodes: at least 3 items per CTA of
    the largest possible grid, more than 256 misses, and a probe of more than one 256-node block."""
    n = planted_nodes(n_sm)
    assert n > 256
    for sh in (S5, S6):
        assert several_items_per_cta(n, sh, n_sm), sh
    assert s8_count(n_sm) >= 2 and several_items_per_cta(s8_count(n_sm), S8, n_sm)
    assert items(n, S5) >= 3 * 8 * n_sm
    assert leaf_grid_max(n_sm) == 8 * n_sm


@pytest.mark.parametrize("policy", [0, 1])
def test_late_tile(policy):
    got = _trade(KINDS["late"].rows, S6, policy)
    assert got is not None and tile_of(leaf_of(got[0], S6)) == tiles(S6) - 1
    assert _trade(KINDS["late"].mutant, S6, policy) is None


def test_ties_across_tiles_chunks_and_lanes():
    """Binpack: the winner uses the later twin for its one branching container; under the mutant the winner is the
    same leaf with the earlier twin, at the same score -- so both leaves were maximal -- and the two leaves lie in
    different tiles / in one tile but different warps / in one warp but different lanes."""
    for name, j, a, b in TIES:
        k = KINDS[name]
        win = _trade(k.rows, S6, 0)
        alt = _trade(k.mutant, S6, 0)
        assert win is not None and alt is not None
        d = [x[0] for x, u in zip(win[0], S6) if u[2] == 0]
        assert d[j] == b, name
        want = [x[0] for x, u in zip(win[0], S6) if u[2] == 0]
        want[j] = a
        assert [x[0] for x, u in zip(alt[0], S6) if u[2] == 0] == want, name
        assert alt[1] == win[1], name
        lw, la = leaf_of(win[0], S6), leaf_of(alt[0], S6)
        assert la < lw
        if name == "tie_tile":
            assert tile_of(la) != tile_of(lw)
        elif name == "tie_chunk":
            assert tile_of(la) == tile_of(lw) and warp_of(la) != warp_of(lw)
        else:
            assert warp_of(la) == warp_of(lw) and chunk_of(la) != chunk_of(lw)


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("sh", [S5, S6, S8], ids=["S5", "S6", "S8"])
def test_neighbouring_misses_disagree(policy, sh):
    e, l = _trade(KINDS["early"].rows, sh, policy), _trade(KINDS["late_low"].rows, sh, policy)
    assert e is not None and l is not None
    le, ll = leaf_of(e[0], sh), leaf_of(l[0], sh)
    assert tile_of(le) < tile_of(ll)
    if policy == 0:
        assert e[1] > l[1]
    if sh is not S8:
        assert tile_of(ll) == tiles(sh) - 1


@pytest.mark.parametrize("policy", [0, 1])
def test_nothing_fits(policy):
    for sh in (S5, S6, S8):
        assert _trade(KINDS["unfit_first"].rows, sh, policy) is None
    for sh in (S6, S8):
        assert _trade(KINDS["unfit_first"].mutant, sh, policy) is not None
    assert _trade(KINDS["unfit_whole"].rows, S5, policy) is None
    assert _trade(KINDS["unfit_whole"].mutant, S5, policy) is not None
    assert _trade(KINDS["unfit_whole"].rows, S6, policy) is not None


@pytest.mark.parametrize("policy", [0, 1])
def test_long_infeasible_prefix(policy):
    k = KINDS["prefix"]
    got = _trade(k.rows, S6, policy)
    assert got is not None
    first = 3 * (1 << 15) + 4 * (1 << 12)
    assert leaf_of(got[0], S6) >= first and first // TILE >= 7
    assert _trade(k.mutant, S6, policy) is None          # every feasible leaf has digit 0 in {3, 4} ...
    alt = [(100, 24), (100, 4), (100, 4), (100, 24), (100, 24), (100, 12), (100, 12), (100, 12)]
    assert _trade(alt, S6, policy) is not None           # ... and, with GPU 3 taken by container 0, digit 1 >= 4:
    blocked = list(k.rows)
    for g in range(4, 8):
        blocked[g] = (100, 4)
    assert _trade(blocked, S6, policy) is None           # nothing fits once GPUs 4..7 take no (1, 8) container


@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("name", ["absent5", "absent6", "absent7"])
def test_absent_digits(policy, name):
    k = KINDS[name]
    for sh in (S5, S6):
        got = _trade(k.rows, sh, policy)
        if got is not None:
            assert all(g < len(k.rows) for a in got[0] for g in a)
        assert got != _trade(k.mutant, sh, policy), (name, sh)


@pytest.mark.parametrize("policy", [0, 1])
def test_every_mutant_changes_the_answer(policy):
    """Each kind's mutant changes the oracle's score, masks or fit under S5, S6 or S8."""
    for name, k in KINDS.items():
        if name == "early":
            continue
        assert any(_trade(k.rows, sh, policy) != _trade(k.mutant, sh, policy) for sh in (S5, S6)), name


def test_planted_cluster_layout():
    n = planted_nodes(132)
    nodes, where = planted_cluster(n)
    assert len(nodes) == n
    for name in KINDS:
        ids = where[name]
        assert len(ids) >= 3, name
        rows = KINDS[name].rows
        assert all(nodes[i][2][0] == [c for c, _ in rows] for i in ids), name
    blocks = set(int(i) // 256 for i in where["late"])
    assert len(blocks) >= 2
    mut, _ = planted_cluster(n, mutate="late_low")
    assert all(mut[i] == nodes[where["early"][0]] for i in where["late_low"])
