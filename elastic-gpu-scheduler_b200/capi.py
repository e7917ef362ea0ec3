"""ctypes binding of include/egs.h (libegs.so).  There is no CPU fallback: loading or
calling fails loudly when the CUDA library is missing or no GPU is present."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence, Tuple

import numpy as np

from . import _build

EGS_MAX_GPUS = 8
EGS_MAX_GPUS_WIDE = 16
EGS_MAX_CONTAINERS = 4
EGS_BINPACK, EGS_SPREAD = 0, 1
(EGS_OK, EGS_ERR_NOFIT, EGS_ERR_NO_OPTION, EGS_ERR_TRANSACT, EGS_ERR_BAD_ARG, EGS_ERR_OVERFLOW_GUARD,
 EGS_ERR_CUDA, EGS_ERR_NO_GPU, EGS_ERR_NO_NODE, EGS_ERR_PANIC, EGS_ERR_COMM) = range(11)
EGS_MODE_AUTO, EGS_MODE_RESCAN, EGS_MODE_ROUNDS = 0, 1, 2
EGS_K_EVALUATE, EGS_K_PASS, EGS_K_SELECT, EGS_K_RESOLVE = 0, 1, 2, 3
EGS_PAD = -(1 << 31)
EGS_HEADROOM_MAX_LIMIT = 1 << 18


def row_width(g_max: int) -> int:
    """EGS_ROW_WIDTH: int32 cells per node row of a handle created with `g_max`."""
    return EGS_MAX_GPUS_WIDE if g_max > EGS_MAX_GPUS else EGS_MAX_GPUS


def mask_dtype(g_max: int):
    """One GPU mask of a handle created with `g_max` (EGS_MASK_BYTES little-endian bytes)."""
    return np.dtype("<u2") if g_max > EGS_MAX_GPUS else np.dtype(np.uint8)


def masks_per_pod(c_max: int) -> int:
    """EGS_MASKS_PER_POD: GPU masks per pod / node of a handle created for pods of up to `c_max` containers."""
    return 8 if c_max > EGS_MAX_CONTAINERS else EGS_MAX_CONTAINERS

# every symbol include/egs.h declares
SYMBOLS = [
    "egs_create", "egs_create_ex", "egs_destroy", "egs_last_error", "egs_status_string", "egs_unit_from_requests",
    "egs_node_set_allocatable", "egs_node_set", "egs_state_load", "egs_state_load_bulk", "egs_state_dump",
    "egs_state_snapshot", "egs_state_restore", "egs_checkpoint_save", "egs_checkpoint_rollback", "egs_checkpoint_drop",
    "egs_filter", "egs_score", "egs_bind", "egs_option_peek", "egs_option_dump", "egs_pod_apply", "egs_node_replay_pod", "egs_pod_cancel",
    "egs_mutations_apply", "egs_schedule_batch_mut", "egs_pod_known", "egs_pod_released", "egs_schedule_batch", "egs_schedule_batch_vec", "egs_schedule_batch_device",
    "egs_schedule_batch_nodes", "egs_headroom", "egs_evict_fit",
    "egs_shard_set", "egs_shard_range", "egs_comm_unique_id", "egs_comm_init", "egs_comm_init_local", "egs_profile_evaluate", "egs_profile_get",
    "egs_profile_reset", "egs_get_stream", "egs_rounds_stats", "egs_mix64",
]


class EgsError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        self.status = status
        super().__init__(f"{where}: egs status {status} {detail}")


_lib = None


def lib_path() -> str:
    return _build.LIBEGS


def load(build: bool = True):
    """dlopen libegs.so (building it with nvcc first when stale)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.build_libegs() if build else _build.LIBEGS
    if os.environ.get("EGS_LIB"):                       # experiments: an alternative build of the same sources
        path = os.path.join(_build.LIBDIR, os.environ["EGS_LIB"])
    if not os.path.exists(path):
        raise RuntimeError(f"{path} is missing: the CUDA extension is required (no CPU fallback)")
    L = C.CDLL(path)
    vp, i32, i64, u64 = C.c_void_p, C.c_int, C.c_int64, C.c_uint64
    L.egs_create.argtypes = [i32, i32, i32, i32, C.POINTER(vp)]
    L.egs_create_ex.argtypes = [i32, i32, i32, i32, i32, C.POINTER(vp)]
    L.egs_destroy.argtypes = [vp]
    L.egs_last_error.argtypes = [vp]; L.egs_last_error.restype = C.c_char_p
    L.egs_status_string.argtypes = [i32]; L.egs_status_string.restype = C.c_char_p
    L.egs_unit_from_requests.argtypes = [i64, i64, vp]
    L.egs_node_set_allocatable.argtypes = [vp, i32, i64, i64]
    L.egs_node_set.argtypes = [vp, i32, i32, i32]
    L.egs_state_load.argtypes = [vp, i32, vp, vp]
    L.egs_state_load_bulk.argtypes = [vp, i32, i32, i32, i32, vp, vp]
    L.egs_state_dump.argtypes = [vp, i32, i32, vp, vp, vp, vp]
    L.egs_state_snapshot.argtypes = [vp]
    L.egs_state_restore.argtypes = [vp]
    L.egs_checkpoint_save.argtypes = [vp]
    L.egs_checkpoint_rollback.argtypes = [vp]
    L.egs_checkpoint_drop.argtypes = [vp]
    L.egs_filter.argtypes = [vp, i32, vp, i32, vp, vp]
    L.egs_score.argtypes = [vp, i32, vp, i32, vp, vp]
    L.egs_bind.argtypes = [vp, i32, i32, vp, u64, vp]
    L.egs_option_peek.argtypes = [vp, i32, i32, vp, vp, vp, vp]
    L.egs_option_dump.argtypes = [vp, i32, vp, i32, i32, vp, vp, vp]
    L.egs_pod_apply.argtypes = [vp, i32, i32, vp, vp, vp, u64]
    L.egs_node_replay_pod.argtypes = [vp, i32, i32, vp, vp, vp, u64]
    L.egs_pod_cancel.argtypes = [vp, i32, i32, vp, vp, vp, u64]
    L.egs_mutations_apply.argtypes = [vp, i32, vp]
    L.egs_schedule_batch_mut.argtypes = [vp, i32, i32, vp, vp, vp, i32, vp, vp] + [vp] * 6
    L.egs_pod_known.argtypes = [vp, u64]
    L.egs_pod_released.argtypes = [vp, u64]
    L.egs_schedule_batch.argtypes = [vp, i32, i32, vp, vp, vp] + [vp] * 6
    L.egs_schedule_batch_vec.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp] + [vp] * 6
    L.egs_schedule_batch_device.argtypes = [vp, i32, i32, vp, vp] + [vp] * 6
    L.egs_schedule_batch_nodes.argtypes = [vp, i32, i32, vp, vp, vp, i32, vp, vp] + [vp] * 6
    L.egs_headroom.argtypes = [vp, i32, vp, vp, i32, i32, vp, i32, vp, vp, vp]
    L.egs_evict_fit.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, vp]
    L.egs_shard_set.argtypes = [vp, i32, i32]
    L.egs_shard_range.argtypes = [i32, i32, i32, C.POINTER(i32), C.POINTER(i32)]
    L.egs_comm_unique_id.argtypes = [vp]
    L.egs_comm_init.argtypes = [vp, vp]
    L.egs_comm_init_local.argtypes = [vp, i32]
    L.egs_profile_evaluate.argtypes = [vp, i32, vp, i32, i32, C.POINTER(C.c_float)]
    L.egs_profile_get.argtypes = [vp, i32, C.POINTER(i64), C.POINTER(C.c_double)]
    L.egs_profile_reset.argtypes = [vp, i32]
    L.egs_rounds_stats.argtypes = [vp, vp]
    L.egs_get_stream.argtypes = [vp, C.POINTER(vp)]
    L.egs_mix64.argtypes = [u64]; L.egs_mix64.restype = u64
    _lib = L
    return L


EGS_MAX_CONTAINERS_APPLY = 8
MUTATION_DTYPE = np.dtype([("kind", "<i4"), ("node_id", "<i4"), ("n_containers", "<i4"), ("pad", "<i4"),
                           ("units", "<i4", (8, 3)), ("n_idx", "i1", (8,)), ("idx", "i1", (8, 8)), ("uid", "<u8")], align=True)
EGS_MUT_ADD, EGS_MUT_FORGET, EGS_MUT_REPLAY = 0, 1, 2


def mutations_array(records) -> np.ndarray:
    """records: [(kind, node_id, req [(core, mem, count)], alloc [[gpu idx]], uid)] -> egs_mutation[]"""
    a = np.zeros(max(1, len(records)), MUTATION_DTYPE)
    for i, (kind, node, req, alloc, uid) in enumerate(records):
        a[i]["kind"], a[i]["node_id"], a[i]["n_containers"], a[i]["uid"] = kind, node, len(req), uid
        for c, u in enumerate(req):
            a[i]["units"][c] = u
            ids = (alloc[c] if alloc and c < len(alloc) and alloc[c] else [])
            a[i]["n_idx"][c] = len(ids)
            for j, g in enumerate(ids):
                a[i]["idx"][c][j] = g
    return a


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def units_array(req: Sequence[Tuple[int, int, int]]) -> np.ndarray:
    a = np.zeros((max(1, len(req)), 3), np.int32)
    for i, u in enumerate(req):
        a[i] = u
    return a


def masks_to_lists(masks, n_containers: int):
    """GPU index lists of the first n_containers masks (up to 8 planes of up to 16 GPUs)."""
    return [[g for g in range(EGS_MAX_GPUS_WIDE) if (int(masks[c]) >> g) & 1] for c in range(n_containers)]


def node_set_words(max_nodes: int) -> int:
    """EGS_NODE_SET_WORDS: 64-bit words of one node set bitmap of a handle with `max_nodes` nodes."""
    return (max_nodes + 63) // 64


def node_sets_array(sets, max_nodes: int) -> np.ndarray:
    """Node sets -> the [n_sets][EGS_NODE_SET_WORDS] uint64 bitmaps of egs_schedule_batch_nodes.  Each set is a bool
    array of max_nodes entries or a list of node ids (bit n & 63 of word n >> 6 admits node n)."""
    out = np.zeros((max(1, len(sets)), node_set_words(max_nodes)), np.uint64)
    for k, s in enumerate(sets):
        a = np.asarray(s)
        if a.dtype == np.bool_:
            if a.shape != (max_nodes,):
                raise ValueError(f"node set {k}: a bool set has max_nodes = {max_nodes} entries, not {a.shape}")
            ids = np.flatnonzero(a)
        else:
            ids = a.astype(np.int64).ravel()
        bits = np.zeros(out.shape[1] * 64, np.uint8)
        bits[ids] = 1                                    # ids at or beyond max_nodes set bits the library refuses
        out[k] = np.packbits(bits, bitorder="little").view("<u8")
    return out


def _alloc_arrays(alloc):
    off, idx = [0], []
    for a in alloc:
        idx.extend(a or [])
        off.append(len(idx))
    return np.array(off, np.int32), np.array(idx + [0], np.int32)


class Egs:
    """One libegs handle == one device.  Method names follow the C ABI.  c_max > 4 makes a sidecar handle
    (egs_create_ex): pods of up to c_max containers, 8 masks per pod."""

    def __init__(self, policy: int, max_nodes: int, g_max: int = 8, device: int = 0, c_max: int = EGS_MAX_CONTAINERS):
        self.L = load()
        self.h = C.c_void_p()
        if c_max == EGS_MAX_CONTAINERS:
            st = self.L.egs_create(policy, max_nodes, g_max, device, C.byref(self.h))
        else:
            st = self.L.egs_create_ex(policy, max_nodes, g_max, c_max, device, C.byref(self.h))
        if st != EGS_OK:
            raise EgsError(st, "egs_create", "(is a CUDA device visible?)")
        self.max_nodes, self.g_max, self.policy, self.c_max = max_nodes, g_max, policy, c_max
        self.row_w, self.mask_dtype, self.n_masks = row_width(g_max), mask_dtype(g_max), masks_per_pod(c_max)

    def close(self):
        if getattr(self, "h", None):
            self.L.egs_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, st: int, where: str):
        if st != EGS_OK:
            raise EgsError(st, where, (self.L.egs_last_error(self.h) or b"").decode())

    # ---- node cache
    def node_set_allocatable(self, node: int, core_alloc: int, mem_alloc: int) -> int:
        return self.L.egs_node_set_allocatable(self.h, node, core_alloc, mem_alloc)

    def node_set(self, node: int, gpu_count: int, mem_total: int) -> int:
        return self.L.egs_node_set(self.h, node, gpu_count, mem_total)

    def state_load(self, node: int, core, mem) -> int:
        c = np.ascontiguousarray(core, np.int32); m = np.ascontiguousarray(mem, np.int32)
        return self.L.egs_state_load(self.h, node, _p(c), _p(m))

    def state_load_bulk(self, node0: int, gpu_count: int, mem_total: int, core: np.ndarray, mem: np.ndarray):
        c = np.ascontiguousarray(core, np.int32); m = np.ascontiguousarray(mem, np.int32)
        self._ck(self.L.egs_state_load_bulk(self.h, node0, c.shape[0], gpu_count, mem_total, _p(c), _p(m)),
                 "egs_state_load_bulk")

    def state_dump(self, node0: int = 0, n: Optional[int] = None):
        n = self.max_nodes - node0 if n is None else n
        core = np.zeros((n, self.row_w), np.int32); mem = np.zeros((n, self.row_w), np.int32)
        gc = np.zeros(n, np.int32); mt = np.zeros(n, np.int32)
        self._ck(self.L.egs_state_dump(self.h, node0, n, _p(core), _p(mem), _p(gc), _p(mt)), "egs_state_dump")
        return core, mem, gc, mt

    def snapshot(self):
        self._ck(self.L.egs_state_snapshot(self.h), "egs_state_snapshot")

    def restore(self):
        self._ck(self.L.egs_state_restore(self.h), "egs_state_restore")

    def checkpoint_save(self):
        """Record the complete scheduler state (egs.h), replacing an earlier checkpoint."""
        self._ck(self.L.egs_checkpoint_save(self.h), "egs_checkpoint_save")

    def checkpoint_rollback(self):
        """Return exactly to the checkpoint, which stays for the next what-if."""
        self._ck(self.L.egs_checkpoint_rollback(self.h), "egs_checkpoint_rollback")

    def checkpoint_drop(self):
        """Forget the checkpoint and free its memory; the current state stays."""
        self._ck(self.L.egs_checkpoint_drop(self.h), "egs_checkpoint_drop")

    def rows(self, node: int):
        core, mem, gc, _ = self.state_dump(node, 1)
        return [(int(core[0, g]), int(mem[0, g])) for g in range(int(gc[0]))]

    # ---- verbs
    def filter(self, node_ids, req) -> np.ndarray:
        ids = None if node_ids is None else np.ascontiguousarray(node_ids, np.int32)
        n = self.max_nodes if ids is None else len(ids)
        out = np.zeros(max(n, 1), np.uint8)
        self._ck(self.L.egs_filter(self.h, n, _p(ids), len(req), _p(units_array(req)), _p(out)), "egs_filter")
        return out[:n]

    def score(self, node_ids, req):
        ids = None if node_ids is None else np.ascontiguousarray(node_ids, np.int32)
        n = self.max_nodes if ids is None else len(ids)
        out = np.zeros(max(n, 1), np.int32)
        st = self.L.egs_score(self.h, n, _p(ids), len(req), _p(units_array(req)), _p(out))
        if st not in (EGS_OK, EGS_ERR_PANIC):
            self._ck(st, "egs_score")
        return st, out[:n]

    def bind(self, node: int, req, uid: int):
        masks = np.zeros(self.n_masks, self.mask_dtype)
        st = self.L.egs_bind(self.h, node, len(req), _p(units_array(req)), uid, _p(masks))
        return st, (masks_to_lists(masks, len(req)) if st == EGS_OK else None)

    def peek(self, node: int, req):
        valid, score = C.c_int32(0), C.c_int32(0)
        masks = np.zeros(self.n_masks, self.mask_dtype)
        self._ck(self.L.egs_option_peek(self.h, node, len(req), _p(units_array(req)), C.byref(valid),
                                        C.byref(score), _p(masks)), "egs_option_peek")
        if not valid.value:
            return None
        return masks_to_lists(masks, len(req)), score.value

    def option_dump(self, req, node0: int = 0, n: Optional[int] = None):
        """Option cache of request `req` on nodes [node0, node0+n): (state u8, score i32, alloc_mask [n, n_masks] of
        mask_dtype: u8, or u16 on a wide handle; n_masks is 4, or 8 on a sidecar handle)."""
        n = self.max_nodes - node0 if n is None else n
        st = np.zeros(max(n, 1), np.uint8); sc = np.zeros(max(n, 1), np.int32)
        am = np.zeros((max(n, 1), self.n_masks), self.mask_dtype)
        self._ck(self.L.egs_option_dump(self.h, len(req), _p(units_array(req)), node0, n, _p(st), _p(sc), _p(am)),
                 "egs_option_dump")
        return st[:n], sc[:n], am[:n]

    def pod_apply(self, node: int, req, alloc, uid: int) -> int:
        off, idx = _alloc_arrays(alloc)
        return self.L.egs_pod_apply(self.h, node, len(req), _p(units_array(req)), _p(off), _p(idx), uid)

    def pod_cancel(self, node: int, req, alloc, uid: int) -> int:
        off, idx = _alloc_arrays(alloc)
        return self.L.egs_pod_cancel(self.h, node, len(req), _p(units_array(req)), _p(off), _p(idx), uid)

    def mutations_apply(self, records) -> int:
        a = mutations_array(records)
        return self.L.egs_mutations_apply(self.h, len(records), _p(a))

    def schedule_batch_mut(self, c_off, units, mut_at, records, uids=None, mode: int = EGS_MODE_AUTO):
        at = np.ascontiguousarray(mut_at, np.int32); a = mutations_array(records)
        return self._batch_call("egs_schedule_batch_mut", (mode,), c_off, units, uids, (len(records), _p(at), _p(a)))

    def pod_known(self, uid: int) -> bool:
        return bool(self.L.egs_pod_known(self.h, uid))

    def pod_released(self, uid: int) -> bool:
        return bool(self.L.egs_pod_released(self.h, uid))

    # ---- batch
    def _batch_out(self, P: int) -> dict:
        """The six per-pod outputs of a batch of P pods, at the handle's mask dtype and plane count."""
        return dict(node=np.zeros(P, np.int32), status=np.zeros(P, np.int32),
                    alloc_mask=np.zeros((P, self.n_masks), self.mask_dtype), fit_count=np.zeros(P, np.int32),
                    fit_digest=np.zeros(P, np.uint64), score_digest=np.zeros(P, np.uint64))

    def _batch_call(self, fn: str, lead, c_off, units, uids, extra=(), out: Optional[dict] = None) -> dict:
        """fn(handle, *lead, P, c_off, units, uids, *extra, the six outputs), its status checked.  Returns the outputs:
        `out`, or the six arrays of _batch_out."""
        out = self._batch_out(len(c_off) - 1) if out is None else out
        c_off = np.ascontiguousarray(c_off, np.int32)
        units = np.ascontiguousarray(units, np.int32)
        u = None if uids is None else np.ascontiguousarray(uids, np.uint64)
        outs = [_p(out[k]) for k in ("node", "status", "alloc_mask", "fit_count", "fit_digest", "score_digest")]
        self._ck(getattr(self.L, fn)(self.h, *lead, len(c_off) - 1, _p(c_off), _p(units), _p(u), *extra, *outs), fn)
        return out

    def schedule_batch(self, c_off: np.ndarray, units: np.ndarray, uids: Optional[np.ndarray] = None,
                       mode: int = EGS_MODE_AUTO):
        return self._batch_call("egs_schedule_batch", (mode,), c_off, units, uids)

    def schedule_batch_nodes(self, c_off: np.ndarray, units: np.ndarray, sets, pod_set=None,
                             uids: Optional[np.ndarray] = None, mode: int = EGS_MODE_AUTO):
        """schedule_batch with a candidate node set per pod (egs_schedule_batch_nodes).  sets: bool arrays of
        max_nodes entries or node-id lists (node_sets_array), or the packed uint64 bitmaps; pod_set: the set of each
        pod (None: every pod uses set 0)."""
        if isinstance(sets, np.ndarray) and sets.dtype == np.uint64 and sets.ndim == 2:
            bm = np.ascontiguousarray(sets)
        else:
            bm = node_sets_array(sets, self.max_nodes)
        ps = None if pod_set is None else np.ascontiguousarray(pod_set, np.int32)
        return self._batch_call("egs_schedule_batch_nodes", (mode,), c_off, units, uids, (len(bm), _p(bm), _p(ps)))

    def schedule_batch_vec(self, c_off: np.ndarray, units: np.ndarray, vec_pods: int, uids: Optional[np.ndarray] = None):
        """schedule_batch + the full fit / score vectors of the first `vec_pods` pods ([vec_pods, N] each)."""
        vec_pods = min(vec_pods, len(c_off) - 1)
        out = self._batch_out(len(c_off) - 1)
        out["vec_fit"] = np.zeros((max(vec_pods, 1), self.max_nodes), np.uint8)
        out["vec_score"] = np.zeros((max(vec_pods, 1), self.max_nodes), np.int32)
        self._batch_call("egs_schedule_batch_vec", (), c_off, units, uids,
                         (vec_pods, _p(out["vec_fit"]), _p(out["vec_score"])), out)
        out["vec_fit"], out["vec_score"] = out["vec_fit"][:vec_pods], out["vec_score"][:vec_pods]
        return out

    def schedule_batch_device(self, c_off: np.ndarray, units: np.ndarray, dptrs: Sequence[int],
                              mode: int = EGS_MODE_AUTO):
        """dptrs: 6 device pointers (node, status, alloc_mask, fit_count, fit_digest, score_digest), 0 = skip."""
        P = len(c_off) - 1
        c_off = np.ascontiguousarray(c_off, np.int32)
        units = np.ascontiguousarray(units, np.int32)
        args = [C.c_void_p(int(p)) if p else None for p in dptrs]
        self._ck(self.L.egs_schedule_batch_device(self.h, mode, P, _p(c_off), _p(units), *args),
                 "egs_schedule_batch_device")

    # ---- capacity
    def headroom(self, shapes, node0: int = 0, n: Optional[int] = None, node_set=None, limit: int = 1 << 16):
        """How many more pods of each shape every node of [node0, node0+n) takes (egs_headroom): per shape a list of
        (core, mem, count) units.  node_set: a bool array of max_nodes entries, a node-id list or one packed bitmap
        (node_sets_array), None for every node.  Returns (count [n_shapes, n] i32, failed [n_shapes, n] i32,
        summary [n_shapes, 4] i64: binds, nodes with a bind, failed binds, nodes stopped by `limit`)."""
        n = self.max_nodes - node0 if n is None else n
        S = len(shapes)
        c_off = np.concatenate([[0], np.cumsum([len(sh) for sh in shapes])]).astype(np.int32)
        units = units_array([u for sh in shapes for u in sh])
        bm = None
        if node_set is not None:
            a = np.asarray(node_set)
            bm = np.ascontiguousarray(a if a.dtype == np.uint64 else node_sets_array([a], self.max_nodes)[0], np.uint64)
        count = np.zeros((S, max(n, 1)), np.int32); failed = np.zeros((S, max(n, 1)), np.int32)
        summary = np.zeros((max(S, 1), 4), np.int64)
        self._ck(self.L.egs_headroom(self.h, S, _p(c_off), _p(units), node0, n, _p(bm), limit, _p(count), _p(failed),
                                     _p(summary)), "egs_headroom")
        return count[:, :n], failed[:, :n], summary[:S]

    # ---- eviction what-if
    def evict_fit(self, req, node_ids, victims=None):
        """Whether pod `req` fits on each node of `node_ids` once that node's victims are forgotten (egs_evict_fit).
        victims: per node a list of (units, alloc, uid) as pod_cancel takes them, None for no victims at all.
        Returns (status [n] i32, score [n] i32, masks [n, n_masks] of mask_dtype)."""
        ids = np.ascontiguousarray(node_ids, np.int32)
        n = len(ids)
        off = recs = None
        if victims is not None:
            off = np.concatenate([[0], np.cumsum([len(v) for v in victims])]).astype(np.int32)
            recs = mutations_array([(EGS_MUT_FORGET, int(node), u, a, uid)
                                    for node, vs in zip(ids, victims) for u, a, uid in vs])
        status = np.zeros(max(n, 1), np.int32); score = np.zeros(max(n, 1), np.int32)
        masks = np.zeros((max(n, 1), self.n_masks), self.mask_dtype)
        self._ck(self.L.egs_evict_fit(self.h, len(req), _p(units_array(req)), n, _p(ids), _p(off), _p(recs),
                                      _p(status), _p(score), _p(masks)), "egs_evict_fit")
        return status[:n], score[:n], masks[:n]

    # ---- sharding / instrumentation
    def shard_set(self, rank: int, world: int):
        self._ck(self.L.egs_shard_set(self.h, rank, world), "egs_shard_set")

    def comm_init(self, uid_bytes: bytes):
        _one_nccl()
        buf = (C.c_uint8 * 128).from_buffer_copy(uid_bytes)
        self._ck(self.L.egs_comm_init(self.h, buf), "egs_comm_init")

    def rounds_stats(self):
        out = np.zeros(8, np.int64)
        self._ck(self.L.egs_rounds_stats(self.h, _p(out)), "egs_rounds_stats")
        keys = ["rounds", "pods", "tracked", "stop_limit", "stop_shape", "stop_tracked_full", "stop_list_dry"]
        return dict(zip(keys, (int(x) for x in out[:7])))

    def stream_ptr(self) -> int:
        out = C.c_void_p()
        self._ck(self.L.egs_get_stream(self.h, C.byref(out)), "egs_get_stream")
        return out.value or 0

    def profile_evaluate(self, req, iters: int = 20, flush_l2: bool = False) -> float:
        ms = C.c_float(0)
        self._ck(self.L.egs_profile_evaluate(self.h, len(req), _p(units_array(req)), iters, int(flush_l2),
                                             C.byref(ms)), "egs_profile_evaluate")
        return ms.value

    def profile_get(self, kernel_id: int):
        n, ms = C.c_int64(0), C.c_double(0)
        self._ck(self.L.egs_profile_get(self.h, kernel_id, C.byref(n), C.byref(ms)), "egs_profile_get")
        return n.value, ms.value

    def profile_reset(self, timing: bool = False):
        self._ck(self.L.egs_profile_reset(self.h, int(timing)), "egs_profile_reset")


def comm_init_local(handles) -> None:
    """In-process shard group over Egs objects (rank r = handles[r]); drive each handle from its own thread."""
    arr = (C.c_void_p * len(handles))(*[h.h for h in handles])
    st = load().egs_comm_init_local(arr, len(handles))
    if st != EGS_OK:
        raise EgsError(st, "egs_comm_init_local")


def _one_nccl():
    """libegs resolves NCCL with dlopen("libnccl.so.2"); importing torch first makes that the
    copy torch bundles, so the process holds a single NCCL."""
    try:
        import torch  # noqa: F401
    except Exception:
        pass


def shard_range(max_nodes: int, rank: int, world: int):
    lo, hi = C.c_int(0), C.c_int(0)
    st = load().egs_shard_range(max_nodes, rank, world, C.byref(lo), C.byref(hi))
    if st != EGS_OK:
        raise EgsError(st, "egs_shard_range")
    return lo.value, hi.value


def comm_unique_id() -> bytes:
    _one_nccl()
    buf = (C.c_uint8 * 128)()
    st = load().egs_comm_unique_id(buf)
    if st != EGS_OK:
        raise EgsError(st, "egs_comm_unique_id")
    return bytes(buf)


def unit_from_requests(core: int, mem: int):
    a = np.zeros(3, np.int32)
    st = load().egs_unit_from_requests(core, mem, _p(a))
    if st != EGS_OK:
        raise EgsError(st, "egs_unit_from_requests")
    return tuple(int(x) for x in a)
