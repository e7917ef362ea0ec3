"""ctypes wrapper of lib/libegs_host.so: the C++ mirror (csrc/host) of the reference's
ResourceScheduler plugin interface (pkg/scheduler/scheduler.go:30-39) with a fake apiserver."""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

from . import _build
from .capi import EGS_MAX_CONTAINERS, EGS_MAX_GPUS

_lib = None


def _load():
    global _lib
    if _lib is None:
        L = C.CDLL(_build.build_host())
        vp, cp, i64 = C.c_void_p, C.c_char_p, C.c_int64
        L.egsh_create.restype = vp; L.egsh_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        L.egsh_destroy.argtypes = [vp]
        L.egsh_register_node.argtypes = [vp, cp, i64, i64]
        L.egsh_register_assumed_pod.argtypes = [vp, cp, vp]
        L.egsh_pod_new.restype = vp; L.egsh_pod_new.argtypes = [cp, cp, cp, cp]
        L.egsh_pod_free.argtypes = [vp]
        L.egsh_pod_add_container.argtypes = [vp, cp, C.c_int, i64, C.c_int, i64]
        L.egsh_pod_set_annotation.argtypes = [vp, cp, cp]
        L.egsh_pod_meta.restype = cp; L.egsh_pod_meta.argtypes = [vp, vp]
        L.egsh_handles.argtypes = [vp]
        L.egsh_assume.restype = cp; L.egsh_assume.argtypes = [vp, vp, C.POINTER(cp), C.c_int]
        L.egsh_score.argtypes = [vp, vp, C.POINTER(cp), C.c_int, C.POINTER(i64)]
        for f in ("egsh_bind",):
            getattr(L, f).restype = cp; getattr(L, f).argtypes = [vp, cp, vp]
        for f in ("egsh_add_pod", "egsh_forget_pod"):
            getattr(L, f).restype = cp; getattr(L, f).argtypes = [vp, vp]
        L.egsh_known_pod.argtypes = [vp, vp]; L.egsh_released_pod.argtypes = [vp, vp]
        L.egsh_status.restype = cp; L.egsh_status.argtypes = [vp]
        L.egsr_new.restype = vp; L.egsr_new.argtypes = [vp]
        L.egsr_free.argtypes = [vp]
        L.egsr_register_pod.argtypes = [vp, vp]
        for f in ("egsr_filter", "egsr_priorities", "egsr_bind"):
            getattr(L, f).restype = cp; getattr(L, f).argtypes = [vp, cp, i64, C.POINTER(C.c_int)]
        _lib = L
    return _lib


class Pod:
    """containers: [(name, {resource: quantity})] with resource in {"core", "memory"}."""

    def __init__(self, name: str, containers, uid: Optional[str] = None, ns: str = "default", node_name: str = "",
                 annotations: Optional[Dict[str, str]] = None):
        self.L = _load()
        self.name, self.ns, self.uid = name, ns, uid or ("uid-" + name)
        self.p = self.L.egsh_pod_new(ns.encode(), name.encode(), self.uid.encode(), node_name.encode())
        for cname, req in containers:
            self.L.egsh_pod_add_container(self.p, cname.encode(), int("core" in req), int(req.get("core", 0)),
                                          int("memory" in req), int(req.get("memory", 0)))
        for k, v in (annotations or {}).items():
            self.L.egsh_pod_set_annotation(self.p, k.encode(), v.encode())

    def __del__(self):
        try:
            if getattr(self, "p", None):
                self.L.egsh_pod_free(self.p)
                self.p = None
        except Exception:
            pass


class CudaUnitScheduler:
    def __init__(self, policy: int, max_nodes: int = 1024, device: int = 0, g_max: int = EGS_MAX_GPUS,
                 c_max: int = EGS_MAX_CONTAINERS):
        """g_max: the widest node; above EGS_MAX_GPUS (up to 16) the handle is wide.  c_max: the widest pod Assume /
        Score / Bind place; above EGS_MAX_CONTAINERS (up to 8, with g_max <= 8) the handle is a sidecar handle."""
        self.L = _load()
        self.h = self.L.egsh_create(policy, max_nodes, device, g_max, c_max)
        if not self.h:
            raise RuntimeError("egsh_create failed (no CUDA device?)")

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.L.egsh_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def register_node(self, name: str, core_alloc: int, mem_alloc: int):
        self.L.egsh_register_node(self.h, name.encode(), core_alloc, mem_alloc)

    def register_assumed_pod(self, node: str, pod: Pod):
        self.L.egsh_register_assumed_pod(self.h, node.encode(), pod.p)

    @staticmethod
    def handles(pod: Pod) -> bool:
        return bool(_load().egsh_handles(pod.p))

    def _names(self, nodes: Sequence[str]):
        arr = (C.c_char_p * len(nodes))(*[n.encode() for n in nodes])
        return arr

    def Assume(self, nodes: Sequence[str], pod: Pod) -> Tuple[List[str], Dict[str, str], Optional[str]]:
        out = self.L.egsh_assume(self.h, pod.p, self._names(nodes), len(nodes)).decode()
        filtered, failed, err = [], {}, None
        for line in out.splitlines():
            parts = line.split("\t")
            if parts[0] == "F":
                filtered.append(parts[1])
            elif parts[0] == "X":
                failed[parts[1]] = parts[2]
            elif parts[0] == "E":
                err = parts[1]
        return filtered, failed, err

    def Score(self, nodes: Sequence[str], pod: Pod) -> List[int]:
        out = (C.c_int64 * max(1, len(nodes)))()
        self.L.egsh_score(self.h, pod.p, self._names(nodes), len(nodes), out)
        return [int(out[i]) for i in range(len(nodes))]

    def Bind(self, node: str, pod: Pod) -> Optional[str]:
        e = self.L.egsh_bind(self.h, node.encode(), pod.p).decode()
        return e or None

    def AddPod(self, pod: Pod) -> Optional[str]:
        return self.L.egsh_add_pod(self.h, pod.p).decode() or None

    def ForgetPod(self, pod: Pod) -> Optional[str]:
        return self.L.egsh_forget_pod(self.h, pod.p).decode() or None

    def KnownPod(self, pod: Pod) -> bool:
        return bool(self.L.egsh_known_pod(self.h, pod.p))

    def ReleasedPod(self, pod: Pod) -> bool:
        return bool(self.L.egsh_released_pod(self.h, pod.p))

    def Status(self) -> str:
        return self.L.egsh_status(self.h).decode()

    def pod_meta(self, pod: Pod):
        ann, lab = {}, {}
        for line in self.L.egsh_pod_meta(self.h, pod.p).decode().splitlines():
            k, a, b = line.split("\t")
            (ann if k == "A" else lab)[a] = b
        return ann, lab


class ExtenderRoutes:
    """The three extender routes end to end over a CudaUnitScheduler: HTTP body in, (status, body) out
    (pkg/routes/routes.go:39-163).  status -1: the reference would panic (body = the panic text)."""

    def __init__(self, sched: CudaUnitScheduler):
        self.L = _load()
        self.s = sched
        self.r = self.L.egsr_new(sched.h)

    def __del__(self):
        try:
            if getattr(self, "r", None):
                self.L.egsr_free(self.r)
                self.r = None
        except Exception:
            pass

    def register_pod(self, pod: Pod):
        self.L.egsr_register_pod(self.r, pod.p)

    def _call(self, f, body: bytes):
        st = C.c_int(0)
        out = f(self.r, body, len(body), C.byref(st))
        return st.value, out.decode()

    def filter(self, body: bytes):
        return self._call(self.L.egsr_filter, body)

    def priorities(self, body: bytes):
        return self._call(self.L.egsr_priorities, body)

    def bind(self, body: bytes):
        return self._call(self.L.egsr_bind, body)
