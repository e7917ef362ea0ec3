"""The oracle's bulk calls (egso_add_nodes, egso_get_rows_many) against the per-node calls they stand for: the same
node ids, GPU counts and rows, and the same answers to a batch afterwards."""
import numpy as np

import oracle_c as oc


def _cluster(seed):
    rng = np.random.default_rng(seed)
    parts = []
    for g in (8, 2, 16, 1, 8):
        n = int(rng.integers(1, 300))
        mt = int(rng.choice([16, 64]))
        core = rng.choice([100, 60, 30, 0], (n, g)).astype(np.int64)
        mem = rng.integers(0, mt + 1, (n, g)).astype(np.int64)
        parts.append((g, mt, core, mem))
    return parts


def _per_node(policy, parts):
    o = oc.OracleC(policy)
    for g, mt, core, mem in parts:
        for i in range(len(core)):
            n = o.add_node(100 * g, mt * g)
            o.set_rows(n, core[i], mem[i])
    return o


def _bulk(policy, parts):
    o = oc.OracleC(policy)
    first = 0
    for g, mt, core, mem in parts:
        assert o.add_nodes(g, mt * g, core, mem) == first
        first += len(core)
    return o


def test_bulk_load_equals_per_node_load():
    for seed in range(4):
        parts = _cluster(seed)
        a, b = _per_node(seed % 2, parts), _bulk(seed % 2, parts)
        n = a.n_nodes
        assert b.n_nodes == n
        ids = np.random.default_rng(seed).permutation(n)
        core, mem, gc = b.rows_many(ids, 16)
        for k, i in enumerate(ids):
            rows = a.rows(int(i))
            assert b.rows(int(i)) == rows and gc[k] == len(rows) == a.gpu_count(int(i))
            assert list(zip(core[k, :len(rows)].tolist(), mem[k, :len(rows)].tolist())) == rows
            assert (core[k, len(rows):] == 0).all() and (mem[k, len(rows):] == 0).all()
        pods = [[(20, 4, 0)], [(0, 0, 1)], [(10, 2, 0), (-1, -1, 0)], [(50, 8, 0)]]
        pick = np.random.default_rng(seed).integers(0, len(pods), 300)
        units = np.array([u for p in pick for u in pods[p]], np.int64)
        c_off = np.concatenate([[0], np.cumsum([len(pods[p]) for p in pick])]).astype(np.int32)
        ra, rb = a.schedule_batch(c_off, units), b.schedule_batch(c_off, units)
        for f in ra:
            assert np.array_equal(ra[f], rb[f]), f
        assert np.array_equal(a.rows_many(ids, 16)[0], b.rows_many(ids, 16)[0])


def test_bulk_load_rejects_bad_gpu_count():
    o = oc.OracleC(0)
    assert o.L.egso_add_nodes(o.h, 4, 17, 1600, None, None) == -1
    assert o.L.egso_add_nodes(o.h, 4, 0, 0, None, None) == -1
    assert o.n_nodes == 0
    assert o.L.egso_add_nodes(o.h, 3, 8, 800, None, None) == 0
    assert o.n_nodes == 3 and o.rows(2) == [(100, 100)] * 8
