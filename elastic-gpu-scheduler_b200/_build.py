"""In-tree builds: libegs.so (CUDA, sm_90a) and libegs_synth.so (plain C harness helper)."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIBEGS = os.path.join(LIBDIR, "libegs.so")
LIBSYNTH = os.path.join(LIBDIR, "libegs_synth.so")

NVCC_FLAGS = (["-DEGS_RESOLVE_PROF"] if os.environ.get("EGS_RESOLVE_PROF") else []) + ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _stale(target: str, sources) -> bool:
    """True when `target` is missing or older than a source or than this file (which holds the flags)."""
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in list(sources) + [os.path.abspath(__file__)])


def nvcc_path() -> str:
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found: libegs cannot be built")
    return p


def _libegs_sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                  glob.glob(os.path.join(CSRC, "*.h")) + [os.path.join(ROOT, "include", "egs.h")])


def build_libegs(force: bool = False, verbose: bool = False) -> str:
    srcs = _libegs_sources()
    if force or _stale(LIBEGS, srcs):
        os.makedirs(LIBDIR, exist_ok=True)
        cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
              ["-o", LIBEGS, os.path.join(CSRC, "egs_api.cu"), "-ldl"]
        subprocess.check_call(cmd)
    return LIBEGS


LIBPROF = os.path.join(LIBDIR, "libegs_prof.so")


def build_prof(force: bool = False) -> str:
    """PROFILING ONLY (tools/gpu_round.sh, tools/prof_sections.py with EGS_LIB=libegs_prof.so): libegs with the
    resolver's clock64 section counters compiled in (-DEGS_RESOLVE_PROF).  Not part of build_all."""
    srcs = _libegs_sources()
    if force or _stale(LIBPROF, srcs):
        os.makedirs(LIBDIR, exist_ok=True)
        flags = [f for f in NVCC_FLAGS if f != "-DEGS_RESOLVE_PROF"]
        subprocess.check_call([nvcc_path(), "-DEGS_RESOLVE_PROF"] + flags + ["-o", LIBPROF, os.path.join(CSRC, "egs_api.cu"), "-ldl"])
    return LIBPROF


def build_synth(force: bool = False) -> str:
    src = os.path.join(CSRC, "egs_synth.c")
    if force or _stale(LIBSYNTH, [src]):
        os.makedirs(LIBDIR, exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-o", LIBSYNTH, src])
    return LIBSYNTH


LIBHOST = os.path.join(LIBDIR, "libegs_host.so")


def build_host(force: bool = False) -> str:
    """C++ mirror of the reference's ResourceScheduler plugin interface over the C ABI."""
    hdir = os.path.join(CSRC, "host")
    srcs = sorted(glob.glob(os.path.join(hdir, "*.cc")) + glob.glob(os.path.join(hdir, "*.h")) +
                  [os.path.join(ROOT, "include", "egs.h")])
    build_libegs(force)
    if force or _stale(LIBHOST, srcs + [LIBEGS]):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", LIBHOST] +
                              sorted(glob.glob(os.path.join(hdir, "*.cc"))) +
                              ["-L" + LIBDIR, "-legs", "-Wl,-rpath,$ORIGIN"])
    return LIBHOST


LIBDEVHOST = os.path.join(LIBDIR, "libegs_devhost.so")


def build_devhost(force: bool = False) -> str:
    """The kernels' integer arithmetic (csrc/egs_device.cuh) compiled for the host: CPU-side tests only."""
    src = os.path.join(CSRC, "host_test", "device_on_host.cu")
    deps = [src, os.path.join(CSRC, "egs_device.cuh"), os.path.join(ROOT, "include", "egs.h")]
    if force or _stale(LIBDEVHOST, deps):
        os.makedirs(LIBDIR, exist_ok=True)
        subprocess.check_call([nvcc_path()] + NVCC_FLAGS + ["-o", LIBDEVHOST, src])
    return LIBDEVHOST


LIBRGEOM = os.path.join(LIBDIR, "libegs_rgeom.so")


def build_rgeom(force: bool = False) -> str:
    """The rounds engine's resolver geometry (mw_geometry, csrc/egs_rounds.cuh) behind a C call: CPU-side tests only."""
    src = os.path.join(CSRC, "host_test", "rounds_geometry_on_host.cu")
    deps = [src] + _libegs_sources()
    if force or _stale(LIBRGEOM, deps):
        os.makedirs(LIBDIR, exist_ok=True)
        subprocess.check_call([nvcc_path()] + NVCC_FLAGS + ["-o", LIBRGEOM, src])
    return LIBRGEOM


LIBPODBOOK = os.path.join(LIBDIR, "libegs_podbook.so")


def build_podbook(force: bool = False) -> str:
    """The uid bookkeeping (csrc/pod_book.h) behind a small C API: CPU-side tests only."""
    src = os.path.join(CSRC, "host_test", "pod_book_on_host.cc")
    deps = [src, os.path.join(CSRC, "pod_book.h"), os.path.join(ROOT, "include", "egs.h")]
    if force or _stale(LIBPODBOOK, deps):
        os.makedirs(LIBDIR, exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-Wall", "-fPIC", "-shared", "-o", LIBPODBOOK, src])
    return LIBPODBOOK


LIBBUFFERS = os.path.join(LIBDIR, "libegs_buffers.so")


def build_buffers(force: bool = False) -> str:
    """The buffer owner (csrc/buffers.h) over a fake allocator behind a small C API: CPU-side tests only."""
    src = os.path.join(CSRC, "host_test", "buffers_on_host.cc")
    deps = [src, os.path.join(CSRC, "buffers.h")]
    if force or _stale(LIBBUFFERS, deps):
        os.makedirs(LIBDIR, exist_ok=True)
        subprocess.check_call([nvcc_path()] + NVCC_FLAGS + ["-o", LIBBUFFERS, src])
    return LIBBUFFERS


SHIM_DOUBLE = os.path.join(ROOT, "integration", "_build", "shim_double")


def build_shim_double(force: bool = False) -> str:
    """C test double of the Go shim (integration/shim_double.c): same libegs calls, same order."""
    src = os.path.join(ROOT, "integration", "shim_double.c")
    build_libegs(force)
    if force or _stale(SHIM_DOUBLE, [src, LIBEGS, os.path.join(ROOT, "include", "egs.h")]):
        os.makedirs(os.path.dirname(SHIM_DOUBLE), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-o", SHIM_DOUBLE, src, "-L" + LIBDIR, "-legs", "-Wl,-rpath," + LIBDIR])
    return SHIM_DOUBLE


def build_all(force: bool = False) -> None:
    build_synth(force)
    build_libegs(force)
    build_host(force)
    build_devhost(force)
    build_rgeom(force)
    build_podbook(force)
    build_buffers(force)
    build_shim_double(force)
