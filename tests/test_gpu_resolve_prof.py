"""The resolver's cycle counters (-DEGS_RESOLVE_PROF build, tools/prof_sections.py): every ticket after the first of a
round is accounted to exactly one kind of hand-over, and the counted build computes what the product build computes.

The profiling build is compiled into a temporary directory and driven from a child process (a process holds one
libegs)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys, ctypes as C
sys.path.insert(0, ROOT); sys.path.insert(0, ROOT + "/oracle")
import numpy as np, egs_b200
w = egs_b200.workloads.config(CFG, n_nodes=NODES, n_pods=PODS)
e = egs_b200.Egs(w.policy, w.n_nodes)
e.state_load_bulk(0, w.gpus, w.mem_total, w.core, w.mem)
got = e.schedule_batch(w.c_off, w.units, mode=2)
out = (C.c_longlong * 32)()
e.L.egs_debug_resolve_prof.argtypes = [C.c_void_p, C.c_void_p]
e.L.egs_debug_resolve_prof(e.h, out)
print(json.dumps({"stats": e.rounds_stats(), "prof": [int(x) for x in out],
                  "out": {f: np.asarray(got[f]).tobytes().hex() for f in ("node", "status", "alloc_mask", "fit_count")}}))
"""


def _run(lib, cfg, nodes, pods):
    env = dict(os.environ)
    if lib:
        env["EGS_LIB"] = lib                                   # absolute: capi joins it onto its lib directory
    else:
        env.pop("EGS_LIB", None)
    code = CHILD.replace("ROOT", repr(ROOT)).replace("CFG", str(cfg)).replace("NODES", str(nodes)).replace("PODS", str(pods))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module")
def prof_lib(tmp_path_factory):
    import egs_b200
    b = egs_b200._build
    lib = str(tmp_path_factory.mktemp("prof") / "libegs_prof.so")
    flags = [f for f in b.NVCC_FLAGS if f != "-DEGS_RESOLVE_PROF"]
    subprocess.check_call([b.nvcc_path(), "-DEGS_RESOLVE_PROF"] + flags + ["-o", lib, os.path.join(b.CSRC, "egs_api.cu"), "-ldl"])
    return lib


@pytest.mark.gpu
@pytest.mark.parametrize("cfg,nodes,pods", [(1, 1000, 10000), (4, 20000, 60000)])
def test_every_ticket_is_accounted_once(prof_lib, cfg, nodes, pods):
    r = _run(prof_lib, cfg, nodes, pods)
    st, v = r["stats"], r["prof"]
    handed, late, kept = v[17], v[21], v[19]
    # per round: every resolved pod but the first took its ticket through one of the three, and so did the pod a
    # tracked-full or list-dry stop was found at
    assert handed + late + kept == st["pods"] - st["rounds"] + st["stop_tracked_full"] + st["stop_list_dry"]
    assert handed > 0 and kept > 0
    assert min(v[16], v[18], v[20]) >= 0 and v[16] >= handed    # a hand-over costs cycles
    base = _run(None, cfg, nodes, pods)
    assert base["stats"] == st
    assert base["out"] == r["out"]
