"""The eviction what-if on the Python oracle (oracle/egs_oracle.py): whether a pending pod fits on a node once the
node's victims are forgotten, found by running the node's own ForgetPod, Assume, Score and Allocate (node.go:61-140)
on a copy of it.  The model egs_evict_fit is tested against."""
import copy

import egs_oracle as po

FRESH_UID = -1                                  # a uid no podsMap holds: the pending pod


def node_evict(na, req, victims):
    """(status, score, alloc) of NodeAllocator `na` for pod `req` after Forget of each victim (units, alloc, uid) in
    order: EGS_ERR_NOFIT, score 0 and alloc None when Assume finds no option; else the option's score, the status of
    Allocate with an unknown uid, and its GPU lists when that is EGS_OK (None otherwise).  `na` is not changed."""
    na = copy.deepcopy(na)
    req = [tuple(u) for u in req]
    for units, alloc, uid in victims:
        units = [tuple(u) for u in units]
        lists = [list(alloc[c]) if alloc and c < len(alloc) and alloc[c] else [] for c in range(len(units))]
        na.forget(units, lists, uid)
    if na.assume(req) is None:
        return po.EGS_ERR_NOFIT, 0, None
    score = na.score(req)
    st, alloc = na.allocate(req, FRESH_UID)
    return st, score, (alloc if st == po.EGS_OK else None)


def applied(pods_map, victims):
    """The victims a node with `pods_map` (uids) forgets, in order: the uid is in the map and no earlier victim of the
    list forgot it -- the podsMap decision ForgetPod takes (node.go:131)."""
    held, out = set(pods_map), []
    for v in victims:
        if v[2] in held:
            held.discard(v[2])
            out.append(v)
    return out
