"""Candidate node sets on the CPU: the oracle driver with per-pod node lists, and the bitmap packing of the binding.
With every node listed, oracle_batch(node_ids=...) is egso_schedule_batch and oracle_batch without lists; a pod's list
keeps it off every other node."""
import numpy as np
import pytest

import oracle_c as oc
from oracle_harness import Cluster, compare_outputs, compare_rows, egs, oracle_batch

PODS = [((30, 4, 0),), ((0, 0, 1),), ((10, 2, 0), (-1, -1, 0)), ((0, 0, 2),)]


def _batch(seed, n_nodes=40, n_pods=120):
    rng = np.random.default_rng(seed)
    nodes = []
    for _ in range(n_nodes):
        g = int(rng.choice([1, 2, 4, 8]))
        core = [int(rng.choice([100, 100, 60, 30])) for _ in range(g)]
        nodes.append((g, 16, (core, [16 if c == 100 else int(rng.integers(4, 17)) for c in core])))
    pick = rng.integers(0, len(PODS), n_pods)
    units = np.array([u for p in pick for u in PODS[p]], np.int32)
    c_off = np.concatenate([[0], np.cumsum([len(PODS[p]) for p in pick])]).astype(np.int32)
    return Cluster(int(seed) & 1, nodes), c_off, units, np.arange(1, n_pods + 1, dtype=np.uint64)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_all_nodes_listed_is_the_batch(seed):
    cl, c_off, units, uids = _batch(seed)
    o_ref, o = cl.oracle(), cl.oracle()
    ref = o_ref.schedule_batch(c_off, units.astype(np.int64), uids)
    every = [np.arange(cl.n_nodes, dtype=np.int32)] * (len(c_off) - 1)
    got = oracle_batch(o, c_off, units, uids, node_ids=every)
    assert (got["alloc_mask"] < 256).all()                      # 8-GPU nodes: the masks fit egso's bytes
    got["alloc_mask"] = got["alloc_mask"].astype(np.uint8)
    compare_outputs(ref, got, f"seed {seed}")
    assert (ref["status"] == 0).any() and (ref["status"] != 0).any()
    compare_rows(_RowsOf(o_ref), o, range(cl.n_nodes))
    compare_outputs(oracle_batch(cl.oracle(), c_off, units, uids), got, f"seed {seed} vs oracle_batch")


def test_lists_keep_pods_on_their_nodes():
    cl, c_off, units, uids = _batch(3)
    P = len(c_off) - 1
    rng = np.random.default_rng(3)
    lists = [np.sort(rng.choice(cl.n_nodes, int(rng.integers(0, cl.n_nodes)), replace=False)).astype(np.int32)
             for _ in range(P)]
    out = oracle_batch(cl.oracle(), c_off, units, uids, node_ids=lists)
    for p in range(P):
        assert out["node"][p] == -1 or out["node"][p] in lists[p]
        assert out["fit_count"][p] <= len(lists[p])
        if len(lists[p]) == 0:
            assert out["status"][p] == 1 and out["fit_count"][p] == 0 and out["fit_digest"][p] == 0


class _RowsOf:
    """An oracle seen through the library's state_dump (rows padded to 8 with EGS_PAD)."""

    def __init__(self, o):
        self.o, self.g_max = o, 8

    def state_dump(self):
        cap = egs().capi
        n = self.o.n_nodes
        core = np.full((n, 8), cap.EGS_PAD, np.int32)
        mem, gc = core.copy(), np.zeros(n, np.int32)
        for i in range(n):
            rows = self.o.rows(i)
            gc[i] = len(rows)
            core[i, :len(rows)], mem[i, :len(rows)] = zip(*rows)
        return core, mem, gc, np.zeros_like(gc)


@pytest.mark.parametrize("max_nodes", [1, 63, 64, 65, 200])
def test_node_sets_array_packs_bits(max_nodes):
    cap = egs().capi
    rng = np.random.default_rng(max_nodes)
    mask = rng.random(max_nodes) < 0.4
    ids = np.flatnonzero(mask)
    a = cap.node_sets_array([mask, ids.tolist(), []], max_nodes)
    assert a.shape == (3, cap.node_set_words(max_nodes)) and a.dtype == np.uint64
    for k in range(2):
        got = [n for n in range(64 * a.shape[1]) if (int(a[k, n >> 6]) >> (n & 63)) & 1]
        assert got == ids.tolist()
    assert not a[2].any()
    with pytest.raises(ValueError):
        cap.node_sets_array([np.ones(max_nodes + 1, bool)], max_nodes)
