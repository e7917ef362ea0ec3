// buffers_on_host.cc -- Buf and grow() (csrc/buffers.h) over a fake allocator behind a C API, so the CPU test suite
// (tests/test_buffers_host.py) can fail any allocation and check that every one is freed exactly once.  Not part of
// libegs.
#include <stdint.h>
#include <string.h>

#include <set>
#include <string>
#include <type_traits>

#include "../buffers.h"

// Host memory standing in for the device.  It fails the fail_at-th allocation, counts frees of pointers it does not
// hold as bad, and logs every call: a = alloc, x = failed alloc, c = copy, s = sync, f = free.
static std::set<void *> g_live;
static long g_allocs = 0, g_fail_at = 0, g_bad_frees = 0;
static std::string g_log;

struct FakeMem {
  static cudaError_t alloc(void **p, size_t bytes) {
    if (++g_allocs == g_fail_at) { g_log += 'x'; return cudaErrorMemoryAllocation; }
    *p = ::operator new(bytes ? bytes : 1);
    g_live.insert(*p);
    g_log += 'a';
    return cudaSuccess;
  }
  static void release(void *p) {
    g_log += 'f';
    if (!g_live.erase(p)) { g_bad_frees++; return; }
    ::operator delete(p);
  }
  static cudaError_t copy(void *dst, const void *src, size_t bytes, cudaStream_t) {
    g_log += 'c';
    memcpy(dst, src, bytes);
    return cudaSuccess;
  }
  static cudaError_t sync(cudaStream_t) { g_log += 's'; return cudaSuccess; }
};

// Three buffers of different element types, grown as one group or one at a time.
struct Trio {
  Buf<int32_t, FakeMem> a;
  Buf<uint8_t, FakeMem> b;
  Buf<uint64_t, FakeMem> c;
};
static Trio *T(void *t) { return (Trio *)t; }

template <class F> static auto on(void *t, int which, F &&f) {
  return which == 0 ? f(T(t)->a) : which == 1 ? f(T(t)->b) : f(T(t)->c);
}

extern "C" {
void egsbuf_fake_reset(long fail_at) { g_allocs = 0; g_fail_at = fail_at; g_bad_frees = 0; g_log.clear(); }
long egsbuf_live() { return (long)g_live.size(); }
long egsbuf_bad_frees() { return g_bad_frees; }
const char *egsbuf_log() { return g_log.c_str(); }

void *egsbuf_new() { return new Trio(); }
void egsbuf_delete(void *t) { delete T(t); }
void *egsbuf_move_new(void *t) { return new Trio(std::move(*T(t))); }                 // t is left empty
void egsbuf_move_assign(void *dst, void *src) { *T(dst) = std::move(*T(src)); }

int egsbuf_grow(void *t, int which, size_t n, int keep) {
  return on(t, which, [&](auto &b) { return (int)grow(nullptr, keep != 0, to(b, n)); });
}
int egsbuf_grow3(void *t, size_t na, size_t nb, size_t nc, int keep) {
  return (int)grow(nullptr, keep != 0, to(T(t)->a, na), to(T(t)->b, nb), to(T(t)->c, nc));
}
size_t egsbuf_cap(void *t, int which) { return on(t, which, [](auto &b) { return b.cap(); }); }
uintptr_t egsbuf_ptr(void *t, int which) { return on(t, which, [](auto &b) { return (uintptr_t)b.get(); }); }
// element i = v + i, over the whole capacity
void egsbuf_fill(void *t, int which, long v) {
  on(t, which, [&](auto &b) { for (size_t i = 0; i < b.cap(); i++) b[i] = (std::remove_reference_t<decltype(b[0])>)(v + (long)i); return 0; });
}
long egsbuf_get(void *t, int which, size_t i) { return on(t, which, [&](auto &b) { return (long)b[i]; }); }
}
