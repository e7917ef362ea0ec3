"""Headroom on the Python oracle (oracle/egs_oracle.py): how many pods of one shape a node still takes when only pods
of that shape arrive, counted by repeating the node's own Assume and Allocate (node.go:61-104) on a copy of it.  The
model egs_headroom is tested against, and which the tests check against a pod-by-pod oracle dry run."""
import copy

import egs_oracle as po


def node_headroom(na, req, limit=None):
    """(ok, failed, capped) of NodeAllocator `na` for request `req`: binds whose Transact succeeds, binds whose
    Transact fails (a stale cached option), and whether `limit` binds stopped a node that still had an option.  `na`
    is not changed."""
    na = copy.deepcopy(na)
    req = [tuple(u) for u in req]
    ok = failed = 0
    while na.assume(req) is not None:
        if limit is not None and ok + failed >= limit:
            return ok, failed, True
        st, _ = na.allocate(req, -1 - ok - failed)          # a uid no podsMap holds
        if st == po.EGS_OK:
            ok += 1
        else:
            assert st == po.EGS_ERR_TRANSACT
            failed += 1
    return ok, failed, False


def allocator(rows, mem_total, policy, req=None, option=None):
    """A NodeAllocator with `rows` [(core, mem)] on GPUs of (100, mem_total), holding `option` = (alloc, score) as
    the cached option of `req` when given."""
    na = po.NodeAllocator(gpus=[po.GPU(c, m, 100, mem_total) for c, m in rows], policy=policy)
    if option is not None:
        alloc, score = option
        na.allocated[na.key([tuple(u) for u in req])] = po.GPUOption(
            request=[tuple(u) for u in req], allocated=[list(a) for a in alloc], score=score)
    return na


def oracle_headroom(o, nodes, policy, req, limit=None):
    """node_headroom of every node of C oracle `o` (oracle_c.OracleC), from its rows and its cached option of `req`.
    nodes: [(gpu_count, mem_total, ...)] as oracle_harness.Cluster holds them, None for an id never set (counts 0).
    Returns three lists: ok, failed, capped."""
    out = ([], [], [])
    for n, nd in enumerate(nodes):
        r = (0, 0, False) if nd is None else node_headroom(allocator(o.rows(n), nd[1], policy, req, o.peek(n, req)),
                                                           req, limit)
        for k in range(3):
            out[k].append(r[k])
    return out
