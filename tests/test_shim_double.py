"""integration/shim_double.c -- the C test double of the Go shim (integration/cuda_scheduler.go) -- replays, per
verb, the C calls the shim makes against libegs.so; every observable answer of seeded scenarios (filter / score /
bind / AddPod / ForgetPod / KnownPod / ReleasedPod / Status, incl. sidecar containers, whole-GPU requests, stale
options, bind failures, unknown nodes) must equal the oracle's."""
import os

import pytest

from scenario import CBackend, make_scenario, run_scenario
from shim_double import ShimDoubleBackend

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "integration", "shim_double.c")


@pytest.mark.gpu
@pytest.mark.parametrize("policy", [0, 1])
@pytest.mark.parametrize("seed", range(12))
def test_shim_call_sequence_vs_oracle(seed, policy):
    nodes, ops = make_scenario(1000 + seed * 2 + policy, max_c=4 if seed % 3 == 0 else 3)
    ref = run_scenario(CBackend(policy), nodes, ops, policy)
    b = ShimDoubleBackend(policy)
    try:
        got = run_scenario(b, nodes, ops, policy)
    finally:
        b.close()
    assert ref == got


def test_double_source_lists_every_shim_call():
    """The double must exercise exactly the entry points the Go shim binds."""
    go = open(os.path.join(ROOT, "integration", "cuda_scheduler.go")).read()
    c = open(SRC).read()
    import re
    used = set(re.findall(r"C\.(egs_[a-z_]+)\(", go))
    assert used, "no cgo calls found"
    missing = {f for f in used if f + "(" not in c and f not in ("egs_last_error", "egs_status_string")}
    assert not missing, f"shim calls not replayed by the double: {missing}"
