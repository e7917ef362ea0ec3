"""The buffer owner -- csrc/buffers.h: Buf and grow() -- compiled for the host over a fake allocator
(csrc/host_test/buffers_on_host.cc) and checked WITHOUT a GPU.  The fake can fail any allocation, counts frees of
pointers it does not hold, and logs every call: a = alloc, x = failed alloc, c = copy, s = sync, f = free."""
import ctypes as C

import pytest

A, B, CC = 0, 1, 2           # the three buffers of a Trio: int32, uint8, uint64


@pytest.fixture(scope="module")
def L():
    import egs_b200
    L = C.CDLL(egs_b200._build.build_buffers())
    vp, sz, i32, lg = C.c_void_p, C.c_size_t, C.c_int, C.c_long
    L.egsbuf_fake_reset.argtypes = [lg]
    L.egsbuf_live.restype = lg
    L.egsbuf_bad_frees.restype = lg
    L.egsbuf_log.restype = C.c_char_p
    L.egsbuf_new.restype = vp
    L.egsbuf_delete.argtypes = [vp]
    L.egsbuf_move_new.argtypes = [vp]
    L.egsbuf_move_new.restype = vp
    L.egsbuf_move_assign.argtypes = [vp, vp]
    L.egsbuf_grow.argtypes = [vp, i32, sz, i32]
    L.egsbuf_grow3.argtypes = [vp, sz, sz, sz, i32]
    L.egsbuf_cap.argtypes = [vp, i32]
    L.egsbuf_cap.restype = sz
    L.egsbuf_ptr.argtypes = [vp, i32]
    L.egsbuf_ptr.restype = C.c_size_t
    L.egsbuf_fill.argtypes = [vp, i32, lg]
    L.egsbuf_get.argtypes = [vp, i32, sz]
    L.egsbuf_get.restype = lg
    return L


@pytest.fixture
def fake(L):
    """Every test starts and must end with no live allocation and no bad free."""
    L.egsbuf_fake_reset(0)
    assert L.egsbuf_live() == 0
    yield L
    assert L.egsbuf_live() == 0
    assert L.egsbuf_bad_frees() == 0


def log(L):
    return L.egsbuf_log().decode()


def state(L, t, which):
    n = L.egsbuf_cap(t, which)
    return L.egsbuf_ptr(t, which), n, [L.egsbuf_get(t, which, i) for i in range(n)]


def test_first_grow_allocates_without_sync(fake):
    L = fake
    t = L.egsbuf_new()
    assert L.egsbuf_grow(t, A, 8, 0) == 0
    assert L.egsbuf_cap(t, A) == 8 and L.egsbuf_ptr(t, A) != 0
    assert log(L) == "a"                          # nothing to free, so nothing to wait for
    L.egsbuf_delete(t)
    assert log(L) == "af"


@pytest.mark.parametrize("keep", [0, 1])
def test_failed_grow_leaves_the_buffer_as_it_was(fake, keep):
    L = fake
    t = L.egsbuf_new()
    assert L.egsbuf_grow(t, A, 8, 0) == 0
    L.egsbuf_fill(t, A, 100)
    before = state(L, t, A)
    L.egsbuf_fake_reset(1)                        # the next allocation fails
    assert L.egsbuf_grow(t, A, 64, keep) != 0
    assert state(L, t, A) == before
    assert log(L) == "x"                          # no copy, no sync, no free
    assert L.egsbuf_live() == 1
    L.egsbuf_delete(t)


def test_preserving_grow_copies_the_old_prefix_then_frees_after_sync(fake):
    L = fake
    t = L.egsbuf_new()
    assert L.egsbuf_grow(t, CC, 5, 0) == 0
    L.egsbuf_fill(t, CC, 1000)
    old = L.egsbuf_ptr(t, CC)
    L.egsbuf_fake_reset(0)
    assert L.egsbuf_grow(t, CC, 12, 1) == 0
    assert L.egsbuf_cap(t, CC) == 12 and L.egsbuf_ptr(t, CC) != old
    assert [L.egsbuf_get(t, CC, i) for i in range(5)] == [1000 + i for i in range(5)]
    assert log(L) == "acsf"                       # alloc, copy, sync, and only then free the old one
    assert L.egsbuf_live() == 1
    L.egsbuf_delete(t)


def test_plain_grow_syncs_before_it_frees(fake):
    L = fake
    t = L.egsbuf_new()
    assert L.egsbuf_grow(t, B, 16, 0) == 0
    L.egsbuf_fake_reset(0)
    assert L.egsbuf_grow(t, B, 32, 0) == 0
    assert log(L) == "asf"
    assert L.egsbuf_cap(t, B) == 32 and L.egsbuf_live() == 1
    L.egsbuf_delete(t)


def test_move_and_destruction_free_each_allocation_once(fake):
    L = fake
    t = L.egsbuf_new()
    assert L.egsbuf_grow3(t, 4, 8, 2, 0) == 0
    ptrs = [L.egsbuf_ptr(t, w) for w in (A, B, CC)]
    u = L.egsbuf_move_new(t)                      # move construction empties the source
    assert [L.egsbuf_ptr(t, w) for w in (A, B, CC)] == [0, 0, 0]
    assert [L.egsbuf_cap(t, w) for w in (A, B, CC)] == [0, 0, 0]
    assert [L.egsbuf_ptr(u, w) for w in (A, B, CC)] == ptrs
    L.egsbuf_delete(t)
    assert L.egsbuf_live() == 3 and "f" not in log(L)
    v = L.egsbuf_new()
    assert L.egsbuf_grow3(v, 1, 1, 1, 0) == 0
    L.egsbuf_fake_reset(0)
    L.egsbuf_move_assign(v, u)                    # v's own three buffers are freed, u's move over
    assert log(L) == "fff" and L.egsbuf_live() == 3
    assert [L.egsbuf_ptr(v, w) for w in (A, B, CC)] == ptrs
    L.egsbuf_move_assign(v, v)                    # self-move keeps the buffers
    assert [L.egsbuf_ptr(v, w) for w in (A, B, CC)] == ptrs and L.egsbuf_live() == 3
    L.egsbuf_delete(u)
    L.egsbuf_delete(v)
    assert L.egsbuf_live() == 0


@pytest.mark.parametrize("fail_at", [2, 3])
@pytest.mark.parametrize("keep", [0, 1])
def test_group_grow_is_all_or_nothing(fake, fail_at, keep):
    L = fake
    t = L.egsbuf_new()
    assert L.egsbuf_grow3(t, 4, 6, 3, 0) == 0
    for w, v in ((A, 10), (B, 20), (CC, 30)):
        L.egsbuf_fill(t, w, v)
    before = [state(L, t, w) for w in (A, B, CC)]
    L.egsbuf_fake_reset(fail_at)
    assert L.egsbuf_grow3(t, 40, 60, 30, keep) != 0
    assert [state(L, t, w) for w in (A, B, CC)] == before
    made = fail_at - 1
    assert log(L) == "a" * made + "x" + "f" * made   # the new ones are freed, no old one is touched
    assert L.egsbuf_live() == 3
    L.egsbuf_fake_reset(0)
    assert L.egsbuf_grow3(t, 40, 60, 30, keep) == 0  # and the group still grows afterwards
    assert [L.egsbuf_cap(t, w) for w in (A, B, CC)] == [40, 60, 30]
    assert log(L) == "aaa" + "ccc" * keep + "s" + "fff"
    if keep:
        assert [L.egsbuf_get(t, B, i) for i in range(6)] == [20 + i for i in range(6)]
    L.egsbuf_delete(t)
