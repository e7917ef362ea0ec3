"""Synthetic clusters and pod batches of BASELINE.json configs 0..4 (SURVEY.md 8d)."""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _build

_lib = None


def _synth():
    global _lib
    if _lib is None:
        _lib = C.CDLL(_build.build_synth())
        _lib.egs_synth_config.argtypes = [C.c_int] + [C.c_void_p] * 5
        _lib.egs_synth_cluster.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        _lib.egs_synth_pods.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return _lib


POLICY_NAMES = {0: "binpack", 1: "spread"}

CONFIG_NAMES = [
    "cfg0: 4 nodes x 2 GPUs, 8 pods gpu-memory, binpack",
    "cfg1: 1000 nodes x 8 GPUs, 10000 pods gpu-core, binpack",
    "cfg2: 10000 nodes x 8 GPUs, 100000 pods core+memory, spread",
    "cfg3: 50000 nodes x 8 GPUs, 500000 multi-container pods, spread",
    "cfg4: 100000 nodes x 8 GPUs, 1000000 pods core+memory, binpack",
]


@dataclass
class Workload:
    cfg: int
    n_nodes: int
    gpus: int
    mem_total: int
    policy: int
    core: np.ndarray      # int32 [n_nodes, gpus]
    mem: np.ndarray       # int32 [n_nodes, gpus]
    c_off: np.ndarray     # int32 [n_pods + 1]
    units: np.ndarray     # int32 [sum C, 3]  (core, mem, count) == egs_unit

    @property
    def n_pods(self) -> int:
        return len(self.c_off) - 1

    def units64(self) -> np.ndarray:
        return self.units.astype(np.int64)

    def prefix(self, n_pods: int) -> "Workload":
        n_pods = min(n_pods, self.n_pods)
        k = int(self.c_off[n_pods])
        return Workload(self.cfg, self.n_nodes, self.gpus, self.mem_total, self.policy, self.core, self.mem,
                        self.c_off[:n_pods + 1].copy(), self.units[:k].copy())


def window(w: "Workload", start: int, n_pods: int) -> "Workload":
    """Pods [start, start + n_pods) of `w` as a batch of their own (same cluster)."""
    end = min(start + n_pods, w.n_pods)
    k0, k1 = int(w.c_off[start]), int(w.c_off[end])
    return Workload(w.cfg, w.n_nodes, w.gpus, w.mem_total, w.policy, w.core, w.mem,
                    (w.c_off[start:end + 1] - k0).astype(np.int32), w.units[k0:k1].copy())


def shapes_of(w: "Workload"):
    """Distinct request shapes of the batch, in order of first appearance: tuples of (core, mem, count)."""
    P = w.n_pods
    if P == 0:
        return []
    n_c = np.diff(w.c_off)
    pods = np.full((P, int(n_c.max()), 3), np.iinfo(np.int32).min, np.int32)   # one padded row of units per pod
    for c in range(pods.shape[1]):
        has = n_c > c
        pods[has, c] = w.units[w.c_off[:-1][has] + c]
    _, first = np.unique(pods.reshape(P, -1), axis=0, return_index=True)
    return [tuple(tuple(int(x) for x in w.units[k]) for k in range(int(w.c_off[p]), int(w.c_off[p + 1])))
            for p in np.sort(first)]


def config(cfg: int, n_nodes: int | None = None, n_pods: int | None = None, policy: int | None = None) -> Workload:
    """Config `cfg` of BASELINE.json; n_nodes / n_pods / policy override the named size
    (the generators are prefix-stable, so a smaller size is a prefix of the full one)."""
    L = _synth()
    vals = [C.c_int() for _ in range(5)]
    if L.egs_synth_config(cfg, *[C.byref(v) for v in vals]) != 0:
        raise ValueError("cfg must be 0..4")
    N, G, M, P, pol = [v.value for v in vals]
    N = N if n_nodes is None else n_nodes
    P = P if n_pods is None else n_pods
    pol = pol if policy is None else policy
    core = np.zeros((N, G), np.int32)
    mem = np.zeros((N, G), np.int32)
    L.egs_synth_cluster(cfg, N, G, M, core.ctypes.data_as(C.c_void_p), mem.ctypes.data_as(C.c_void_p))
    c_off = np.zeros(P + 1, np.int32)
    units = np.zeros((3 * P + 1, 3), np.int32)
    k = L.egs_synth_pods(cfg, P, c_off.ctypes.data_as(C.c_void_p), units.ctypes.data_as(C.c_void_p))
    return Workload(cfg, N, G, M, pol, core, mem, c_off, units[:k].copy())
