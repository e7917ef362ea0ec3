"""Batches for the rounds engine (EGS_MODE_ROUNDS): pods over a list of distinct shapes, arriving all at the front or
trickling in, on a cluster; and the check of one batch's egs_rounds_stats."""
import numpy as np

from oracle_harness import Cluster

STOPS = ["stop_limit", "stop_shape", "stop_tracked_full", "stop_list_dry"]
RSMAX = 96                                   # shapes per round set


def pod_picks(rng, shapes, n_pods, arrival):
    """Pod -> shape index.  "front": every shape in the first pods, then uniform picks.  "trickle": six phases; phase
    i picks among a window of 64 shapes that moves on by 40 shapes a phase (cyclically), each shape's first pod at
    the start of its first phase.  Above 96 shapes a round that runs into the next phase meets more than 96 distinct
    shapes, so the host-formed sets hold part of the batch's shapes and change from round to round."""
    n = len(shapes)
    if arrival == "front":
        rest = rng.integers(0, n, max(0, n_pods - n))
        return np.concatenate([np.arange(min(n, n_pods)), rest]).astype(np.int64)
    assert arrival == "trickle"
    w, span, seen, out = min(64, n), n_pods // 6, set(), []
    for i in range(6):
        window = [(40 * i + t) % n for t in range(w)]
        new = [s for s in window if s not in seen]
        seen.update(new)
        m = n_pods - len(out) if i == 5 else span
        out += new + [window[int(j)] for j in rng.integers(0, w, m - len(new))]
    assert len(seen) == n and len(out) == n_pods
    return np.array(out, np.int64)


class Batch:
    """Pod p has shape shapes[pick[p]]; c_off / units in the layout of egs_schedule_batch."""

    def __init__(self, policy, nodes, shapes, pick):
        self.cluster, self.shapes = Cluster(policy, nodes), shapes
        self.n_nodes, self.n_pods = len(nodes), len(pick)
        c_off, units = [0], []
        for s in pick:
            units.extend(shapes[int(s)])
            c_off.append(len(units))
        self.c_off = np.array(c_off, np.int32)
        self.units = np.array(units, np.int32).reshape(-1, 3)


def distinct_shapes(b):
    """Distinct shapes of the batch as the library sees them (workloads.shapes_of's counting)."""
    seen, out = set(), []
    for p in range(b.n_pods):
        u = tuple(tuple(int(x) for x in b.units[k]) for k in range(int(b.c_off[p]), int(b.c_off[p + 1])))
        if u not in seen:
            seen.add(u); out.append(u)
    return out


def stats_delta(s1, s0):
    return {k: s1[k] - s0[k] for k in s1}


def check_paths(d, n_shapes, n_pods):
    """egs_rounds_stats delta of one batch: every round has exactly one stop reason, every pod was resolved, and
    "shape outside the round set" occurs exactly when the host forms the sets."""
    assert sum(d[k] for k in STOPS) == d["rounds"], d
    assert d["pods"] == n_pods, d
    if n_shapes > RSMAX:
        assert d["stop_shape"] > 0, d
    else:
        assert d["stop_shape"] == 0, d
