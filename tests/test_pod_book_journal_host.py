"""The checkpoint of the uid bookkeeping -- csrc/pod_book.h's undo journal -- compiled for the host
(csrc/host_test/pod_book_on_host.cc) and checked WITHOUT a GPU: seeded sequences of operations, a save, more operations
and a rollback, repeated from the same checkpoint.  After every rollback the book must equal a model made of three
plain sets as it stood at the save, on every (node, uid) the sequence touched, and keep the same hash_uid_max."""
import copy
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
    L.egspb_checkpoint.argtypes = [vp]
    L.egspb_rollback.argtypes = [vp]
    L.egspb_drop_checkpoint.argtypes = [vp]
    L.egspb_hash_uid_max.argtypes = [vp]; L.egspb_hash_uid_max.restype = u64
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


class Journaled:
    """A PodBook and the model driven by the same operations, with a checkpoint: save() keeps a copy of the model,
    the library-uid counter and the book's hash_uid_max; rollback() returns the book and the model to them."""

    def __init__(self, PB):
        self.L, self.b, self.m = PB, PB.egspb_create(), Model()
        self.next_uid = AUTO
        self.touched = set()
        self.saved = None
        self.stats = dict(ops=0, runs=0, rollbacks=0)

    def close(self):
        self.L.egspb_free(self.b)

    # ---- the operations of test_pod_book_host.py's model, each checked against it as it runs
    def run(self, node, status):
        n = len(node)
        uids = list(range(self.next_uid, self.next_uid + n))
        nd, sd = np.array(node, np.int32), np.array(status, np.int32)
        self.L.egspb_add_run(self.b, self.next_uid, n, nd.ctypes.data, sd.ctypes.data)
        self.m.batch(uids, node, status)
        self.next_uid += n
        self.touched.update(uids)
        self.stats["runs"] += 1

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
        assert (rc, [int(c) for c in cancels[:n.value]]) == self.m.account(kind, node, uid, fail), (kind, node, hex(uid))
        self.touched.add(uid)

    def drop(self, node0, n):
        self.L.egspb_drop_nodes(self.b, node0, n)
        self.m.drop(node0, n)

    def clear(self):
        self.L.egspb_clear(self.b)
        self.m.clear()

    # ---- the checkpoint
    def save(self):
        self.L.egspb_checkpoint(self.b)
        self.saved = (copy.deepcopy(self.m), self.next_uid, int(self.L.egspb_hash_uid_max(self.b)))

    def rollback(self):
        self.L.egspb_rollback(self.b)
        m, self.next_uid, hmax = self.saved
        self.m = copy.deepcopy(m)
        assert int(self.L.egspb_hash_uid_max(self.b)) == hmax, "hash_uid_max after the rollback"
        self.stats["rollbacks"] += 1

    def drop_checkpoint(self):
        self.L.egspb_drop_checkpoint(self.b)
        self.saved = None

    def check(self, where=""):
        for u in sorted(self.touched | {0, 999, self.next_uid, self.next_uid + 7, AUTO + (1 << 40)}):
            assert bool(self.L.egspb_in_pod_maps(self.b, u)) == (u in self.m.maps), (where, "podMaps", hex(u))
            assert bool(self.L.egspb_released(self.b, u)) == (u in self.m.released), (where, "released", hex(u))
            for n in range(NN):
                assert bool(self.L.egspb_in_pods_map(self.b, n, u)) == ((n, u) in self.m.pods), (where, "podsMap", n, hex(u))

    def __call__(self, op, *args, **kw):
        getattr(self, op)(*args, **kw)
        self.stats["ops"] += 1
        self.check((op, args))


def _random_ops(p, rng, n_ops, clear_p=0.03):
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
        elif k < 1 - clear_p:
            if rng.random() < 0.5:
                p("drop", 0, NN)
            else:
                n0 = node()
                p("drop", n0, rng.randint(1, NN - n0))
        else:
            p("clear")


def test_erased_run_and_its_neighbours_come_back(PB):
    """A forget empties a run in the middle, a reload empties podsMap bits of the others, clear() empties the book;
    each rollback puts every run back where it was, with its bits and counts."""
    p = Journaled(PB)
    p("run", [0, 1], [OK, OK])                           # run A
    U = p.next_uid
    p("run", [2], [OK])                                  # run B: one pod, erased below
    p("run", [3, -1], [OK, NOFIT])                       # run C
    p.save()
    p("account", FORGET, 2, U)                           # B loses both bits and is erased; U is released
    p("account", FORGET, 2, U)
    p("bind", 1, AUTO, True, OK)                         # a key of A outside its home: the hash set
    p("drop", 0, NN)                                     # every podsMap bit of A and C goes; C keeps podMaps
    p("account", FORGET, -1, AUTO + 3)
    p.rollback(); p.check("first rollback")
    p("clear")
    p("run", [0], [OK])
    p.rollback(); p.check("second rollback")
    p.drop_checkpoint()
    p("account", FORGET, 3, AUTO + 3)
    p.check("after drop")
    p.close()


@pytest.mark.parametrize("seed", range(30))
def test_random_sequences_roll_back_to_the_save(PB, seed):
    rng = random.Random(1000 + seed)
    p = Journaled(PB)
    for _ in range(3):                                   # three checkpoints, each replacing the last
        _random_ops(p, rng, rng.randint(0, 60))
        p.save()
        for _ in range(3):                               # several what-ifs from the same checkpoint
            _random_ops(p, rng, rng.randint(1, 50), clear_p=0.05)
            p.rollback()
            p.check("after rollback")
    p.drop_checkpoint()
    _random_ops(p, rng, 20)                              # the book works on without a checkpoint
    p.close()
    assert p.stats["rollbacks"] == 9
