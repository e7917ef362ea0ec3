"""The uid bookkeeping -- csrc/pod_book.h: NodeAllocator.podsMap and the scheduler's podMaps / releasedPodMap, with
library-assigned uids kept in per-batch runs -- compiled for the host (csrc/host_test/pod_book_on_host.cc) and
checked WITHOUT a GPU against a model made of three plain sets, one rule per line of the reference."""
import ctypes as C
import random

import numpy as np
import pytest

OK, NOFIT, NO_OPTION, TRANSACT, BAD_ARG = 0, 1, 2, 3, 4
ADD, FORGET, REPLAY = 0, 1, 2
AUTO = 1 << 63                  # the first library-assigned uid
NN = 4                          # nodes


@pytest.fixture(scope="module")
def PB():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_podbook())
    vp, i32, u64 = C.c_void_p, C.c_int, C.c_uint64
    L.egspb_create.restype = vp
    L.egspb_free.argtypes = [vp]
    L.egspb_add_run.argtypes = [vp, u64, i32, vp, vp]
    L.egspb_add_batch.argtypes = [vp, vp, i32, vp, vp]
    L.egspb_record_bind.argtypes = [vp, i32, u64, i32, i32, i32]
    L.egspb_account.argtypes = [vp, i32, i32, u64, i32, vp, vp]
    L.egspb_drop_nodes.argtypes = [vp, i32, i32]
    L.egspb_clear.argtypes = [vp]
    L.egspb_in_pods_map.argtypes = [vp, i32, u64]
    L.egspb_in_pod_maps.argtypes = [vp, u64]
    L.egspb_released.argtypes = [vp, u64]
    return L


class Model:
    """podsMap of every NodeAllocator as (node, uid) pairs (node.go:16), podMaps and releasedPodMap
    (scheduler.go:47-49)."""

    def __init__(self):
        self.pods, self.maps, self.released = set(), set(), set()

    def batch(self, uids, node, status):
        for u, n, s in zip(uids, node, status):
            if n >= 0:
                self.pods.add((n, u))                    # node.go:150, before Transact: a failed Transact keeps it
                if s == OK:
                    self.maps.add(u)                     # scheduler.go:224

    def bind(self, node, uid, had_entry, status):
        if had_entry:
            self.pods.add((node, uid))                   # Allocate found an option: node.go:149-150
        if status == OK:
            self.maps.add(uid)                           # scheduler.go:224

    def account(self, kind, node, uid, fail):
        """-> (status, cancel arguments of the row updates made).  A failing row update ends the record."""
        if kind == FORGET:                               # ForgetPod scheduler.go:247-267
            calls = []
            if node >= 0 and (node, uid) in self.pods:   # node.go:131
                calls.append(1)
                if fail:
                    return BAD_ARG, calls
                self.pods.discard((node, uid))           # node.go:136
            if uid in self.maps:                         # scheduler.go:261-264
                self.maps.discard(uid)
                self.released.add(uid)
            return OK, calls
        if kind == ADD and uid in self.maps:             # scheduler.go:239-241
            return OK, []
        calls = []
        if (node, uid) not in self.pods:                 # node.go:149
            calls.append(0)
            if fail:
                return BAD_ARG, calls
            self.pods.add((node, uid))                   # node.go:150
        if kind == ADD:
            self.maps.add(uid)                           # scheduler.go:243
        return OK, calls

    def drop(self, node0, n):                            # a reloaded node gets a fresh NodeAllocator (node.go:42-50)
        self.pods = {k for k in self.pods if not node0 <= k[0] < node0 + n}

    def clear(self):
        self.pods, self.maps, self.released = set(), set(), set()


class Pair:
    """A PodBook and the model, driven by the same operations and compared after each one."""

    def __init__(self, PB):
        self.L, self.b, self.m = PB, PB.egspb_create(), Model()
        self.next_uid = AUTO
        self.touched = set()

    def close(self):
        self.L.egspb_free(self.b)

    def run(self, node, status):
        """a batch with library-assigned uids; returns them"""
        n = len(node)
        uids = list(range(self.next_uid, self.next_uid + n))
        nd, sd = np.array(node, np.int32), np.array(status, np.int32)
        self.L.egspb_add_run(self.b, self.next_uid, n, nd.ctypes.data, sd.ctypes.data)
        self.m.batch(uids, node, status)
        self.next_uid += n
        self.touched.update(uids)
        return uids

    def batch(self, uids, node, status):
        ud, nd, sd = np.array(uids, np.uint64), np.array(node, np.int32), np.array(status, np.int32)
        self.L.egspb_add_batch(self.b, ud.ctypes.data, len(uids), nd.ctypes.data, sd.ctypes.data)
        self.m.batch(uids, node, status)
        self.touched.update(uids)

    def bind(self, node, uid, had_entry, status):
        known = self.L.egspb_in_pods_map(self.b, node, uid)          # as egs_bind asks before k_bind
        self.L.egspb_record_bind(self.b, node, uid, int(had_entry), known, status)
        self.m.bind(node, uid, had_entry, status)
        self.touched.add(uid)

    def account(self, kind, node, uid, fail=False):
        n, cancels = C.c_int(0), np.zeros(4, np.int32)
        rc = self.L.egspb_account(self.b, kind, node, uid, int(fail), C.byref(n), cancels.ctypes.data)
        want = self.m.account(kind, node, uid, fail)
        assert (rc, [int(c) for c in cancels[:n.value]]) == want, (kind, node, hex(uid), fail)
        self.touched.add(uid)
        return rc

    def drop(self, node0, n):
        self.L.egspb_drop_nodes(self.b, node0, n)
        self.m.drop(node0, n)

    def clear(self):
        self.L.egspb_clear(self.b)
        self.m.clear()

    def check(self, where=""):
        for u in sorted(self.touched | {0, 999, self.next_uid, self.next_uid + 7, AUTO + (1 << 40)}):
            assert bool(self.L.egspb_in_pod_maps(self.b, u)) == (u in self.m.maps), (where, "podMaps", hex(u))
            assert bool(self.L.egspb_released(self.b, u)) == (u in self.m.released), (where, "released", hex(u))
            for n in range(NN):
                assert bool(self.L.egspb_in_pods_map(self.b, n, u)) == ((n, u) in self.m.pods), (where, "podsMap", n, hex(u))

    def __call__(self, op, *args, **kw):
        r = getattr(self, op)(*args, **kw)
        self.check((op, args))
        return r


def test_auto_uid_rebound_on_another_node_then_forgotten(PB):
    """Bind sets podMaps[U] again without looking (scheduler.go:224); ForgetPod on the second node then deletes U
    (scheduler.go:261-264) while the first node's podsMap keeps it."""
    p = Pair(PB)
    U, = p("run", [0], [OK])
    p("bind", 1, U, True, OK)
    assert p("account", FORGET, 1, U) == OK
    assert not PB.egspb_in_pod_maps(p.b, U) and PB.egspb_released(p.b, U)
    assert PB.egspb_in_pods_map(p.b, 0, U) and not PB.egspb_in_pods_map(p.b, 1, U)
    p.close()


def test_auto_uid_traps(PB):
    """An auto uid bound, added and replayed on its own node and on another; forgotten twice; re-added after the
    forget; reloads in between, full and partial."""
    p = Pair(PB)
    U, V, W, X = p("run", [0, 1, -1, 2], [OK, TRANSACT, NOFIT, OK])
    p("bind", 0, U, True, OK)                            # own node: already in podsMap
    p("account", ADD, 0, U)                              # known: no-op
    p("account", REPLAY, 0, U)                           # in podsMap: no row update
    p("account", REPLAY, 1, U)                           # another node: row update, podsMap of node 1
    p("account", ADD, 3, V)                              # V failed its Transact: not in podMaps
    p("account", FORGET, 0, U)
    p("account", FORGET, 0, U)                           # twice: nothing left to forget
    p("account", FORGET, 1, U)
    p("account", ADD, 0, U)                              # re-added after the forget
    p("drop", 0, NN)                                     # full reload
    p("account", FORGET, 0, U)                           # podsMap gone with the node; podMaps kept U
    p("account", ADD, 0, U)
    p("bind", 2, X, True, OK)                            # own node, after a reload in between
    p("drop", 1, 1)                                      # partial reload
    p("account", REPLAY, 1, V)
    p("account", FORGET, -1, V)                          # empty NodeName
    p("account", FORGET, 2, X, fail=True)                # the row update fails: the record ends there
    p("account", FORGET, 2, X)
    p("bind", 3, W, False, NO_OPTION)
    p("bind", 3, W, True, TRANSACT)
    p("account", ADD, 3, W, fail=True)
    p("account", ADD, 3, W)
    p("drop", 0, NN)
    p("account", REPLAY, 0, U)
    p("clear")
    p("account", ADD, 0, U)
    p.close()


def test_caller_uid_inside_a_later_run(PB):
    """A caller-given uid that a later batch assigns again: the keys it had stay visible."""
    p = Pair(PB)
    U = p.next_uid + 1
    p("batch", [U], [2], [OK])
    p("bind", 3, U + 1, True, TRANSACT)
    p("run", [2, 3, 3], [NOFIT, TRANSACT, OK])
    p("account", FORGET, 2, U)
    p("account", FORGET, 3, U + 1)
    p.close()


def _random_ops(p, rng, n_ops):
    def uid():
        r = rng.random()
        if p.touched and r < 0.7:
            return rng.choice(sorted(p.touched))
        if r < 0.9:
            return rng.randint(1, 6)
        return p.next_uid + rng.randint(0, 3)            # an auto uid before its batch assigns it

    node = lambda: rng.randint(0, NN - 1)
    for _ in range(n_ops):
        k = rng.random()
        if k < 0.15:
            n = rng.randint(1, 6)
            p("run", [rng.choice([-1, -1] + list(range(NN))) for _ in range(n)],
              [rng.choice([OK, OK, NOFIT, TRANSACT]) for _ in range(n)])
        elif k < 0.25:
            us = list(dict.fromkeys(uid() for _ in range(rng.randint(1, 4))))
            p("batch", us, [rng.choice([-1] + list(range(NN))) for _ in us], [rng.choice([OK, NOFIT, TRANSACT]) for _ in us])
        elif k < 0.45:
            had = rng.random() < 0.8
            p("bind", node(), uid(), had, rng.choice([OK, OK, NOFIT, TRANSACT]) if had else NO_OPTION)
        elif k < 0.9:
            kind = rng.choice([ADD, FORGET, REPLAY])
            nd = rng.choice([-1, node()]) if kind == FORGET else node()
            p("account", kind, nd, uid(), fail=rng.random() < 0.15)
        elif k < 0.97:
            if rng.random() < 0.5:
                p("drop", 0, NN)
            else:
                n0 = node()
                p("drop", n0, rng.randint(1, NN - n0))
        else:
            p("clear")


@pytest.mark.parametrize("seed", range(40))
def test_random_sequences_equal_model(PB, seed):
    rng = random.Random(seed)
    p = Pair(PB)
    _random_ops(p, rng, 150)
    p.close()
