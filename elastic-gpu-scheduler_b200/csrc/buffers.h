// buffers.h -- the one owner of libegs's device and pinned host memory (host code only).
//
// Buf<T, Mem> owns one allocation of cap() elements of T and frees it exactly once, in its destructor.  Buffers are
// (re)allocated by grow() alone, which makes every new allocation before it frees an old one: a grow that fails
// leaves every buffer -- pointer, capacity and contents -- as it was.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include <algorithm>
#include <tuple>
#include <utility>

// Mem policies: alloc / release one allocation; copy (for a grow that keeps the contents) and sync on a stream.
struct DeviceMem {
  static cudaError_t alloc(void **p, size_t bytes) { return cudaMalloc(p, bytes); }
  static void release(void *p) { cudaFree(p); }
  static cudaError_t copy(void *dst, const void *src, size_t bytes, cudaStream_t s) {
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, s);
  }
  static cudaError_t sync(cudaStream_t s) { return cudaStreamSynchronize(s); }
};
struct PinnedMem {
  static cudaError_t alloc(void **p, size_t bytes) { return cudaMallocHost(p, bytes); }
  static void release(void *p) { cudaFreeHost(p); }
  static cudaError_t copy(void *dst, const void *src, size_t bytes, cudaStream_t s) {
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToHost, s);
  }
  static cudaError_t sync(cudaStream_t s) { return cudaStreamSynchronize(s); }
};

template <class T, class Mem>
class Buf {
 public:
  using mem = Mem;
  Buf() = default;
  Buf(Buf &&o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
  Buf &operator=(Buf &&o) noexcept { Buf(std::move(o)).swap(*this); return *this; }
  Buf(const Buf &) = delete;
  Buf &operator=(const Buf &) = delete;
  ~Buf() { if (p_) Mem::release(p_); }

  T *get() const { return p_; }
  operator T *() const { return p_; }
  T *operator->() const { return p_; }
  size_t cap() const { return n_; }                              // in elements
  void swap(Buf &o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); }

  // A new allocation of n elements replaces the buffer, which is freed at once: for a Buf no stream can still use.
  cudaError_t alloc(size_t n) {
    void *p = nullptr;
    const cudaError_t e = Mem::alloc(&p, n * sizeof(T));
    if (e == cudaSuccess) { Buf b; b.p_ = (T *)p; b.n_ = n; swap(b); }
    return e;
  }
  // The first n elements of o, copied on s.
  cudaError_t copy_from(const Buf &o, size_t n, cudaStream_t s) {
    return n ? Mem::copy(p_, o.p_, n * sizeof(T), s) : cudaSuccess;
  }

 private:
  T *p_ = nullptr;
  size_t n_ = 0;
};

template <class T> using DeviceBuf = Buf<T, DeviceMem>;
template <class T> using PinnedBuf = Buf<T, PinnedMem>;

template <class B> struct Want { B &buf; size_t n; };
template <class B> Want<B> to(B &buf, size_t n) { return Want<B>{buf, n}; }

// Replaces each listed buffer by a new allocation of its own element count, all or none: every new allocation is
// made first, and they replace the old buffers only when all of them succeeded.  With keep, each old buffer's
// elements (as many as fit) are copied into its successor on s first.  An old allocation is freed only after s has
// drained, since kernels and copies on s may still use it (every policy synchronises a stream the same way).
template <class... B>
cudaError_t grow(cudaStream_t s, bool keep, Want<B>... w) {
  using First = std::tuple_element_t<0, std::tuple<B...>>;
  std::tuple<B...> next;                     // freed on return: the new allocations after a failure, else the old ones
  return std::apply([&](B &...nb) {
    cudaError_t e = cudaSuccess;
    ((e = e == cudaSuccess ? nb.alloc(w.n) : e), ...);
    if (keep) ((e = e == cudaSuccess ? nb.copy_from(w.buf, std::min(w.n, w.buf.cap()), s) : e), ...);
    if (e == cudaSuccess && (w.buf.cap() || ...)) e = First::mem::sync(s);
    if (e == cudaSuccess) (w.buf.swap(nb), ...);
    return e;
  }, next);
}
