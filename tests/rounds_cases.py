"""Seeded clusters, shapes and batches for the rounds model (tests/rounds_model.py) against the Python oracle, and the
replay that compares the two batch by batch.  The over-totals shapes also feed the GPU tests of that regime."""
import numpy as np

import egs_oracle as po


def model_cluster(rng, n_nodes):
    """(core_alloc, mem_alloc, rows or None): 1-8 GPUs of 16-80 MiB, about half of the nodes partly used."""
    nodes = []
    for _ in range(n_nodes):
        g = int(rng.choice([1, 2, 4, 8]))
        m = int(rng.choice([16, 40, 80]))
        rows = None
        if rng.integers(0, 2):
            rows = ([int(rng.choice([100, 100, 60, 30, 0])) for _ in range(g)], [int(rng.integers(0, m + 1)) for _ in range(g)])
        nodes.append((100 * g, m * g, rows))
    return nodes


def model_shapes(rng, n, mono):
    """n shapes of 1-3 containers: fractional, whole-GPU and (unless mono) sentinel units."""
    out = []
    for _ in range(n):
        units = []
        for _ in range(int(rng.integers(1, 4))):
            k = rng.integers(0, 10)
            if k == 0 and not mono:
                units.append((-1, -1, 0))
            elif k == 1:
                units.append((0, 0, int(rng.integers(1, 3))))
            else:
                units.append((int(rng.choice([0, 5, 10, 25, 50])), int(rng.integers(1, 12)), 0))
        out.append(tuple(units))
    return out


def model_scenario(seed):
    """(rng, K, T, RS, D, nodes, shapes): a cluster and shapes at a tiny list depth K / tracked table T / shape set RS
    and 1-3 shards D, so that every early stop fires; monotone shapes (no sentinel) when seed % 3 == 0.  The caller
    draws its pods from rng."""
    rng = np.random.default_rng(seed)
    K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
    nodes = model_cluster(rng, int(rng.integers(3, 40)))
    shapes = model_shapes(rng, int(rng.integers(1, 7)), seed % 3 == 0)
    return rng, K, T, RS, D, nodes, shapes


def model_batches(rng, shapes):
    """Three batches of 20-159 pods, run one after another on the same state."""
    return [[shapes[int(i)] for i in rng.integers(0, len(shapes), int(rng.integers(20, 160)))] for _ in range(3)]


def fast_regime(seed):
    """(K, T, D, nodes, pods): single-container fractional shapes only, the benchmark's monotone rounds."""
    rng = np.random.default_rng(5000 + seed)
    K, T, D = int(rng.choice([1, 2, 4])), int(rng.choice([2, 3, 4, 6])), int(rng.choice([1, 2, 3]))
    nodes = model_cluster(rng, int(rng.integers(6, 30)))
    shapes = [((int(rng.choice([5, 10, 25, 50])), int(rng.integers(1, 12)), 0),) for _ in range(int(rng.integers(1, 5)))]
    pods = [shapes[int(i)] for i in rng.integers(0, len(shapes), 200)]
    return K, T, D, nodes, pods


def load_nodes(nodes, *scheds):
    """The same nodes, in order, on every scheduler given (models and the oracle)."""
    for core, mem, rows in nodes:
        (n,) = {s.add_node(core, mem) for s in scheds}
        for s in scheds if rows else ():
            s.set_rows(n, *rows)


def check_batch(m, o, pods, uid, tag):
    """The batch through the model and pod by pod through the oracle (uids from `uid` on): the six outputs of every pod
    equal.  Returns the oracle's per-pod results."""
    got = m.schedule_batch(pods)
    rs = []
    for p, (s, g) in enumerate(zip(pods, got)):
        r = o.schedule_one(list(s), uid + p)
        assert g == {k: r[k] for k in ("node", "status", "alloc", "fit_count", "fit_digest", "score_digest")}, tag + (p,)
        rs.append(r)
    return rs


def replay(m, o, batches, tag, uid=0):
    """Each batch through the model and the oracle: outputs, rows and option caches equal after every batch, and no
    option the model memoises as UNFIT fits the oracle's rows.  Returns the number of whole-GPU pods the oracle bound
    on a node that had a GPU above its totals when the batch began."""
    n_regime = 0
    for b, pods in enumerate(batches):
        over = [o.nodes[n] is not None and any(g.core_avail > g.core_total or g.mem_avail > g.mem_total for g in o.nodes[n].gpus)
                for n in range(len(m.nodes))]
        for s, r in zip(pods, check_batch(m, o, pods, uid, tag + (b,))):
            n_regime += r["status"] == po.EGS_OK and over[r["node"]] and any(u[2] > 0 for u in s)
        uid += len(pods)
        for n in range(len(m.nodes)):
            assert m.rows(n) == o.rows(n), tag + (b, n)
        for s in set(pods):
            for n in range(len(m.nodes)):
                e = m.tables[s][n]
                opt = o.nodes[n].allocated.get(tuple(s)) if o.nodes[n] is not None else None
                assert (e.st == 1) == (opt is not None), tag + (b, s, n, e.st)
                if opt is not None:
                    assert (e.score, e.alloc) == (opt.score, opt.allocated), tag + (b, s, n)
                if e.st == 2:
                    assert po.trade(o.nodes[n].gpus, po.RATERS[m.policy], list(s)) is None, tag + (b, s, n, "unfit fits")
    return n_regime


# ------------------------------------------------------------------------------------------------ GPUs above their totals
# A GPU can hold more than its totals: a container without a GPU request (the (-1, -1) sentinel) ADDS 1 to the GPU it
# lands on (gpu.go:36-37), ForgetPod gives back what a failed AddPod never took (node.go:149-150, gpu.go:177-191), and a
# loaded row may be anything up to the int32 guard.  Such a GPU is not free for a whole-GPU container (gpu.go:193-202)
# until a fractional bind brings it down to exactly its totals -- so a round whose requests are all >= 0 can still turn
# an option that did not fit into one that fits.
SIDECAR, WHOLE1, FRAC11 = ((-1, -1, 0),), ((0, 0, 1),), ((1, 1, 0),)
MINIMAL = [[SIDECAR], [WHOLE1, FRAC11, WHOLE1]]   # one node, one GPU of 16 MiB: (101, 17) after batch 1
OVER = (0, 0, 1, 1, 1, 2, 3)   # how far a GPU starts above its totals, per row


def over_totals_cluster(rng, n_nodes):
    """Nodes of 1, 2 or 4 GPUs whose every GPU is at or just above its totals: core 100..103, memory mt..mt+3, most
    of them 1 above."""
    nodes = []
    for _ in range(n_nodes):
        g, mt = int(rng.choice([1, 2, 4])), int(rng.choice([8, 16]))
        rows = ([100 + int(rng.choice(OVER)) for _ in range(g)], [mt + int(rng.choice(OVER)) for _ in range(g)])
        nodes.append((100 * g, mt * g, rows))
    return nodes


def over_totals_shapes(rng, n):
    """n distinct shapes, every request >= 0: whole-GPU containers of count 1 or 2 (alone or with one fractional
    container), and 1-3 fractional containers of 0-3 core and 0-3 MiB, mostly 0-1 -- small enough to bring a GPU
    just above its totals back to them.  The first two are WHOLE1 and FRAC11, which undoes the most common excess."""
    def frac():
        while True:
            u = (int(rng.choice(OVER)), int(rng.choice(OVER)), 0)
            if u[0] or u[1]:
                return u
    out = [WHOLE1, FRAC11]
    while len(out) < n:
        if rng.integers(0, 2):
            sh = ((0, 0, int(rng.integers(1, 3))),) + ((frac(),) if rng.integers(0, 3) == 0 else ())
        else:
            sh = tuple(frac() for _ in range(int(rng.integers(1, 4))))
        if sh not in out:
            out.append(sh)
    return out


def over_totals_scenario(seed):
    """(policy, K, T, RS, D, nodes, batches): three batches on one state at the tiny list depth / tracked table /
    shape set of model_scenario."""
    rng = np.random.default_rng(9000 + seed)
    K, T, RS, D = int(rng.choice([1, 2, 3, 8])), int(rng.choice([2, 3, 5, 64])), int(rng.choice([1, 2, 4, 32])), int(rng.choice([1, 2, 3]))
    nodes = over_totals_cluster(rng, int(rng.integers(3, 24)))
    shapes = over_totals_shapes(rng, int(rng.integers(2, 7)))
    batches = [[shapes[int(i)] for i in rng.integers(0, len(shapes), int(rng.integers(20, 120)))] for _ in range(3)]
    return seed % 2, K, T, RS, D, nodes, batches
