"""Every decision of the full-size benchmark batches against the oracle.

The plain oracle Assumes every node for every pod, too slow for whole batches of configs 2 to 4; the indexed driver
(egso_schedule_batch_indexed, pinned to the plain one by test_oracle_indexed_host.py) makes the same decisions in
seconds.  Each test compares all six per-pod outputs of every pod with it, then the rows of every node and the option
cache of every shape on every node.  The oracle's answer for a (config, policy) is computed once per module."""
import os
import time

import numpy as np
import pytest
import torch

from oracle_harness import FIELDS, Cluster, compare_caches, compare_outputs, compare_rows, egs
from shard_groups import ShardGroup

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def answer():
    """answer(cfg, policy=None) -> (workload, the indexed oracle's outputs, the oracle after the batch), once per
    module for each (config, policy)."""
    memo = {}

    def get(cfg, policy=None):
        if (cfg, policy) not in memo:
            w = egs().workloads.config(cfg, policy=policy)
            o = Cluster.of_workload(w).oracle()
            t0 = time.perf_counter()
            ref = o.schedule_batch_indexed(w.c_off, w.units64(), threads=os.cpu_count() or 1)
            print(f"indexed oracle cfg{cfg} policy {w.policy}: {time.perf_counter() - t0:.1f} s")
            memo[(cfg, policy)] = (w, ref, o)
        return memo[(cfg, policy)]
    return get


def check_state(e, w, o):
    compare_rows(e, o, range(w.n_nodes))
    compare_caches(e, o, egs().workloads.shapes_of(w), range(w.n_nodes), unfit_check=True)


# ------------------------------------------------------------------------------------------------ engines
@pytest.mark.parametrize("cfg,policy", [(1, None), (2, None), (3, None), (4, None), (4, 1), (3, 0)])
def test_rounds_engine_whole_batch(answer, cfg, policy):
    """Configs 1 to 4 under their own policies, config 4 under spread and config 3 under binpack."""
    w, ref, o = answer(cfg, policy)
    e = Cluster.of_workload(w).handle()
    got = e.schedule_batch(w.c_off, w.units, mode=egs().capi.EGS_MODE_ROUNDS)
    compare_outputs(ref, got, f"cfg{cfg} policy {w.policy}, rounds")
    check_state(e, w, o)
    e.close()


@pytest.mark.parametrize("cfg", [1, 2, 4])
def test_rescan_engine_whole_batch(answer, cfg):
    """One launch per pod: a million launches on config 4, about 10 s on an H100 (700 W)."""
    w, ref, o = answer(cfg)
    e = Cluster.of_workload(w).handle()
    got = e.schedule_batch(w.c_off, w.units, mode=egs().capi.EGS_MODE_RESCAN)
    compare_outputs(ref, got, f"cfg{cfg}, rescan")
    check_state(e, w, o)
    e.close()


# ------------------------------------------------------------------------------------------------ the benchmark's path
@pytest.mark.parametrize("cfg", [1, 2, 3, 4])
def test_resident_steps_as_the_benchmark_runs_them(answer, cfg):
    """bench.py's timed step: rows loaded in bulk and snapshotted, the batch through egs_schedule_batch_device into
    torch device buffers, then egs_state_restore and the same batch again.  Both steps equal the oracle, so a restored
    handle answers like a fresh one."""
    w, ref, o = answer(cfg)
    eg = egs()
    e = eg.Egs(w.policy, w.n_nodes, 8, 0)
    e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
    e.snapshot()
    dev, P = torch.device("cuda", 0), w.n_pods
    bufs = [torch.empty(P, dtype=torch.int32, device=dev), torch.empty(P, dtype=torch.int32, device=dev),
            torch.empty((P, 4), dtype=torch.uint8, device=dev), torch.empty(P, dtype=torch.int32, device=dev),
            torch.empty(P, dtype=torch.int64, device=dev), torch.empty(P, dtype=torch.int64, device=dev)]
    for step in range(2):
        for b in bufs:
            b.fill_(-1 if b.dtype != torch.uint8 else 0xAB)
        torch.cuda.synchronize()
        if step:
            e.restore()
        e.schedule_batch_device(w.c_off, w.units, [b.data_ptr() for b in bufs])
        torch.cuda.synchronize()
        got = {f: b.cpu().numpy() for f, b in zip(FIELDS, bufs)}
        got["fit_digest"], got["score_digest"] = got["fit_digest"].view(np.uint64), got["score_digest"].view(np.uint64)
        compare_outputs(ref, got, f"cfg{cfg}, resident step {step}")
    check_state(e, w, o)
    e.close()


# ------------------------------------------------------------------------------------------------ shard groups
@pytest.mark.parametrize("cfg,world", [(3, 4), (4, 8)])
def test_shard_group_at_the_benchmark_world_size(answer, cfg, world):
    """An in-process shard group of `world` handles on one device, as the benchmark shards config 3 (4 ranks) and
    config 4 (8 ranks): every rank's outputs equal the oracle's, and each rank's rows over its own node range equal
    the oracle's rows there."""
    w, ref, o = answer(cfg)
    cl = Cluster.of_workload(w)
    rounds = egs().capi.EGS_MODE_ROUNDS
    with ShardGroup(cl, world) as g:
        outs = g.each(lambda r, h: h.schedule_batch(w.c_off, w.units, mode=rounds))
        for r, out in enumerate(outs):
            compare_outputs(ref, out, f"cfg{cfg}, world {world}, rank {r}")
        for r in range(world):
            lo, hi = g.ranges[r]
            core, mem = g.on(r, lambda _r, h: h.state_dump(lo, hi - lo)[:2])
            ocore, omem, _ = o.rows_many(np.arange(lo, hi), core.shape[1])
            assert np.array_equal(core[:, :w.gpus], ocore[:, :w.gpus]) and \
                np.array_equal(mem[:, :w.gpus], omem[:, :w.gpus]), f"cfg{cfg}, world {world}: rows of shard {r}"

