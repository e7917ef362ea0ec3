// egs_api.cu -- host side of libegs: the C ABI of include/egs.h over the device-resident
// SoA node/GPU cache.  No CPU fallback exists: every verb runs a CUDA kernel or fails.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "egs_kernels.cuh"
#include "egs_rounds.cuh"
#include "pod_book.h"

struct Shape { int C; egs_unit u[EGS_C]; };

// Pinned host buffer holding (node[n], status[n]) of a batch.  Recycled through egs_handle::pin_pool: cudaMallocHost /
// cudaFreeHost cost milliseconds and synchronise the device -- too much for a small batch on the extender's path.
struct PinBuf { int32_t *p = nullptr; size_t cap = 0; };   // cap in int32 elements
struct PendingBatch {           // results of a batch whose uid bookkeeping is applied lazily
  int n; uint64_t uid0; std::vector<uint64_t> uids; int32_t *h_node, *h_status; PinBuf buf; cudaEvent_t done;
};

struct egs_handle {
  int policy = 0, max_nodes = 0, n_pad = 0, g_max = 0, device = 0, n_sm = 0;
  int row_w = EGS_G, mask_b = 1;          // EGS_ROW_WIDTH(g_max), EGS_MASK_BYTES(g_max)
  int rank = 0, world = 1, lo = 0, hi = 0;
  cudaStream_t stream = nullptr;
  int32_t *d_core = nullptr, *d_mem = nullptr, *d_mem_total = nullptr;
  int32_t *d_snap_core = nullptr, *d_snap_mem = nullptr, *d_snap_total = nullptr;
  std::vector<int32_t> snap_gpu_count, snap_mem_total;
  std::vector<int32_t> h_gpu_count, h_mem_total;
  // option tables
  int slot_cap = 0;
  uint8_t *d_st = nullptr; int32_t *d_sc = nullptr; uint8_t *d_al = nullptr;
  std::vector<Shape> shapes;
  std::vector<char> slot_cold;            // option table of the slot holds only OPT_ABSENT (nothing evaluated yet)
  std::unordered_map<std::string, int> shape_ids;
  struct ShapeCacheEnt { uint64_t h; int slot; };
  std::vector<ShapeCacheEnt> shape_cache = std::vector<ShapeCacheEnt>(1024, ShapeCacheEnt{0, -1});   // open addressing
  // reference bookkeeping that never reaches the device
  PodBook book;                                                 // podsMap / podMaps / releasedPodMap
  std::vector<PendingBatch> pending;                            // batches whose results have not reached the book
  std::vector<PinBuf> pin_pool;                                 // idle pinned result buffers (at most PIN_POOL_MAX)
  uint64_t next_uid = 0x8000000000000000ull;
  // scratch
  Partial *d_partials = nullptr; unsigned int *d_ticket = nullptr; int32_t *d_result = nullptr;
  int32_t *h_result = nullptr;                                  // pinned
  int32_t *d_ids = nullptr; uint8_t *d_fit = nullptr; int32_t *d_score = nullptr; size_t gather_cap = 0;
  void *h_stage = nullptr; size_t h_stage_cap = 0;              // pinned staging
  // eval scratch (profile)
  uint8_t *d_ev_fit = nullptr; int32_t *d_ev_score = nullptr; uint8_t *d_ev_gpu = nullptr; void *d_flush = nullptr;
  // batch outputs
  int32_t *d_o_node = nullptr, *d_o_status = nullptr, *d_o_fit = nullptr; uint8_t *d_o_alloc = nullptr;
  unsigned long long *d_o_fd = nullptr, *d_o_sd = nullptr; int out_cap = 0;
  void *d_ops = nullptr; int32_t *d_group_off = nullptr; size_t ops_cap = 0;   // egs_mutations_apply: ApplyOp<row_w>[]
  uint8_t *d_vec_fit = nullptr; int32_t *d_vec_score = nullptr; size_t vec_cap = 0; int vec_pods = 0;   // egs_schedule_batch_vec
  // profiling
  int64_t k_launches[EGS_K_COUNT] = {0}; double k_ms[EGS_K_COUNT] = {0}; int timing = 0;
  RoundsState rounds;
  std::mutex mu;
  std::string err;
};

#define CK(h, call)                                                                      \
  do {                                                                                   \
    cudaError_t e_ = (call);                                                             \
    if (e_ != cudaSuccess) {                                                             \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                     \
      return EGS_ERR_CUDA;                                                               \
    }                                                                                    \
  } while (0)
#define TRY(expr) do { int rc_ = (expr); if (rc_ != EGS_OK) return rc_; } while (0)

static int fail(egs_handle *h, int code, const char *msg) { h->err = msg; return code; }

// The one place the row width picks a kernel instantiation: f(std::integral_constant<int, G>()) with G the handle's
// row width, 8 or 16.
template <class F>
static int by_width(const egs_handle *h, F &&f) {
  return h->row_w == 16 ? f(std::integral_constant<int, 16>()) : f(std::integral_constant<int, EGS_G>());
}
static bool is_wide(const egs_handle *h) { return h->row_w > EGS_G; }

// Packed option masks (container c at bits [G*c, G*c + G)) -> EGS_MAX_CONTAINERS little-endian masks of mask_b bytes.
static void put_masks(const egs_handle *h, uint64_t masks, uint8_t *out) {
  for (int c = 0; c < EGS_C; c++)
    for (int b = 0; b < h->mask_b; b++) out[c * h->mask_b + b] = (uint8_t)(masks >> (h->row_w * c + 8 * b));
}

static int ensure_stage(egs_handle *h, size_t bytes) {
  if (bytes <= h->h_stage_cap) return EGS_OK;
  if (h->h_stage) cudaFreeHost(h->h_stage);
  h->h_stage = nullptr; h->h_stage_cap = 0;
  size_t cap = std::max(bytes, (size_t)1 << 20);
  CK(h, cudaMallocHost(&h->h_stage, cap));
  h->h_stage_cap = cap;
  return EGS_OK;
}

static OptTable table(egs_handle *h, int slot) {
  OptTable t;
  t.plane = (size_t)h->n_pad;
  t.st = h->d_st + (size_t)slot * h->n_pad;
  t.sc = h->d_sc + (size_t)slot * h->n_pad;
  t.al = h->d_al + (size_t)slot * EGS_C * h->n_pad * h->mask_b;
  return t;
}

static int grow_slots(egs_handle *h, int need) {
  if (need <= h->slot_cap) return EGS_OK;
  int cap = std::max(need, std::max(16, h->slot_cap * 2));
  uint8_t *st; int32_t *sc; uint8_t *al;
  size_t np = (size_t)h->n_pad, al_plane = np * EGS_C * h->mask_b;
  CK(h, cudaMalloc(&st, np * cap));
  CK(h, cudaMalloc(&sc, np * cap * sizeof(int32_t)));
  CK(h, cudaMalloc(&al, al_plane * cap));
  CK(h, cudaMemsetAsync(st, OPT_ABSENT, np * cap, h->stream));
  if (h->slot_cap) {
    CK(h, cudaMemcpyAsync(st, h->d_st, np * h->slot_cap, cudaMemcpyDeviceToDevice, h->stream));
    CK(h, cudaMemcpyAsync(sc, h->d_sc, np * h->slot_cap * sizeof(int32_t), cudaMemcpyDeviceToDevice, h->stream));
    CK(h, cudaMemcpyAsync(al, h->d_al, al_plane * h->slot_cap, cudaMemcpyDeviceToDevice, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    cudaFree(h->d_st); cudaFree(h->d_sc); cudaFree(h->d_al);
  }
  h->d_st = st; h->d_sc = sc; h->d_al = al; h->slot_cap = cap;
  return EGS_OK;
}

static int check_units(int C, const egs_unit *u, int max_c = EGS_C) {
  if (C < 1 || C > max_c || !u) return EGS_ERR_BAD_ARG;
  for (int i = 0; i < C; i++) {
    if (u[i].count < 0) return EGS_ERR_BAD_ARG;
    if (u[i].core < -1 || u[i].mem < -1) return EGS_ERR_BAD_ARG;
    if (u[i].core > EGS_MAX_CORE_LOAD || u[i].mem > EGS_MAX_MEM_PER_GPU) return EGS_ERR_OVERFLOW_GUARD;
  }
  return EGS_OK;
}

// request -> option-table slot.  The reference keys its cache on sha256(String())[0:8]
// (allocate.go:30-33); the unit tuple is the same key up to a 32-bit prefix collision.
static inline uint64_t shape_hash(int C, const egs_unit *u) {
  uint64_t x = 0x9E3779B97F4A7C15ull * (uint64_t)C;
  for (int i = 0; i < C; i++) {
    x = mix64(x ^ (((uint64_t)(uint32_t)u[i].core << 32) | (uint32_t)u[i].mem));
    x ^= (uint64_t)(uint32_t)u[i].count * 0xD6E8FEB86659FD93ull;
  }
  return x | 1;
}

static int intern_slow(egs_handle *h, int C, const egs_unit *u, int *slot);

// hot entry: one hash + one probe per pod (a batch of 10^6 pods re-uses a handful of shapes)
static inline int intern(egs_handle *h, int C, const egs_unit *u, int *slot) {
  if (C >= 1 && C <= EGS_C && u) {
    const uint64_t hv = shape_hash(C, u);
    const size_t mask = h->shape_cache.size() - 1;
    for (size_t i = hv & mask, n = 0; n < 8; i = (i + 1) & mask, n++) {
      const auto &e = h->shape_cache[i];
      if (e.slot < 0) break;
      if (e.h == hv) {
        const Shape &sh = h->shapes[e.slot];
        if (sh.C == C && memcmp(sh.u, u, sizeof(egs_unit) * C) == 0) { *slot = e.slot; return EGS_OK; }
      }
    }
  }
  TRY(intern_slow(h, C, u, slot));
  if (h->shapes.size() * 4 > h->shape_cache.size()) h->shape_cache.assign(h->shape_cache.size() * 4, egs_handle::ShapeCacheEnt{0, -1});
  const uint64_t hv = shape_hash(C, u);
  const size_t mask = h->shape_cache.size() - 1;
  for (size_t i = hv & mask, n = 0; n < 8; i = (i + 1) & mask, n++)
    if (h->shape_cache[i].slot < 0) { h->shape_cache[i] = egs_handle::ShapeCacheEnt{hv, *slot}; break; }
  return EGS_OK;
}

static int intern_slow(egs_handle *h, int C, const egs_unit *u, int *slot) {
  TRY(check_units(C, u));
  std::string key((const char *)&C, sizeof C);
  key.append((const char *)u, sizeof(egs_unit) * C);
  auto it = h->shape_ids.find(key);
  if (it != h->shape_ids.end()) { *slot = it->second; return EGS_OK; }
  int s = (int)h->shapes.size();
  TRY(grow_slots(h, s + 1));
  Shape sh; sh.C = C; memset(sh.u, 0, sizeof sh.u); memcpy(sh.u, u, sizeof(egs_unit) * C);
  h->shapes.push_back(sh);
  h->slot_cold.push_back(1);
  h->shape_ids.emplace(key, s);
  *slot = s;
  return EGS_OK;
}

static bool is_single(int C, const egs_unit *u) { return C == 1 && u[0].count == 0 && u[0].core >= 0 && u[0].mem >= 0; }

constexpr size_t PIN_POOL_MAX = 4;
static void pin_put(egs_handle *h, PinBuf b) {
  if (!b.p) return;
  if (h->pin_pool.size() < PIN_POOL_MAX) h->pin_pool.push_back(b); else cudaFreeHost(b.p);
}

static int flush_pending(egs_handle *h) {
  for (auto &b : h->pending) {
    CK(h, cudaEventSynchronize(b.done));
    if (b.uids.empty()) h->book.add_run(b.uid0, b.n, b.h_node, b.h_status);     // library-assigned uids
    else h->book.add_batch(b.uids.data(), b.n, b.h_node, b.h_status);
    pin_put(h, b.buf); cudaEventDestroy(b.done);
  }
  h->pending.clear();
  return EGS_OK;
}

struct Guard {
  egs_handle *h; std::lock_guard<std::mutex> lk;
  explicit Guard(egs_handle *hh) : h(hh), lk(hh->mu) { cudaSetDevice(hh->device); }
};

static int pin_get(egs_handle *h, size_t n, PinBuf *out) {
  int best = -1;                                                // smallest idle buffer that is large enough
  for (size_t i = 0; i < h->pin_pool.size(); i++)
    if (h->pin_pool[i].cap >= n && (best < 0 || h->pin_pool[i].cap < h->pin_pool[(size_t)best].cap)) best = (int)i;
  if (best >= 0) { *out = h->pin_pool[(size_t)best]; h->pin_pool.erase(h->pin_pool.begin() + best); return EGS_OK; }
  PinBuf b; b.cap = std::max(n, (size_t)4096);
  CK(h, cudaMallocHost(&b.p, b.cap * sizeof(int32_t)));
  *out = b;
  return EGS_OK;
}

// ------------------------------------------------------------------------------- lifecycle
extern "C" int egs_create(int policy, int max_nodes, int g_max, int device, egs_handle **out) {
  if (!out || max_nodes < 1 || g_max < 1 || g_max > EGS_MAX_GPUS_WIDE || (policy != EGS_BINPACK && policy != EGS_SPREAD))
    return EGS_ERR_BAD_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1 || device < 0 || device >= ndev) return EGS_ERR_CUDA;
  egs_handle *h = new egs_handle();
  h->policy = policy; h->max_nodes = max_nodes; h->g_max = g_max; h->device = device;
  h->row_w = EGS_ROW_WIDTH(g_max); h->mask_b = EGS_MASK_BYTES(g_max);
  h->n_pad = (max_nodes + 1023) / 1024 * 1024;
  h->lo = 0; h->hi = max_nodes;
  h->h_gpu_count.assign(max_nodes, 0); h->h_mem_total.assign(max_nodes, 0);
  auto boot = [&]() -> int {
    CK(h, cudaSetDevice(device));
    CK(h, cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
    CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    size_t rows = (size_t)h->n_pad * h->row_w * sizeof(int32_t);
    CK(h, cudaMalloc(&h->d_core, rows));
    CK(h, cudaMalloc(&h->d_mem, rows));
    CK(h, cudaMalloc(&h->d_mem_total, (size_t)h->n_pad * sizeof(int32_t)));
    CK(h, cudaMemsetAsync(h->d_mem_total, 0, (size_t)h->n_pad * sizeof(int32_t), h->stream));
    // EGS_PAD == 0x80000000: fill through a pinned pattern-free path (memset is per byte)
    std::vector<int32_t> pad((size_t)h->n_pad * h->row_w, EGS_PAD);
    CK(h, cudaMemcpy(h->d_core, pad.data(), rows, cudaMemcpyHostToDevice));
    CK(h, cudaMemcpy(h->d_mem, pad.data(), rows, cudaMemcpyHostToDevice));
    int nblk = (h->n_pad + PASS_THREADS - 1) / PASS_THREADS;
    CK(h, cudaMalloc(&h->d_partials, sizeof(Partial) * (size_t)nblk));
    CK(h, cudaMalloc(&h->d_ticket, sizeof(unsigned int) * 4));
    CK(h, cudaMemsetAsync(h->d_ticket, 0, sizeof(unsigned int) * 4, h->stream));
    CK(h, cudaMalloc(&h->d_result, sizeof(int32_t) * 16));
    CK(h, cudaMallocHost(&h->h_result, sizeof(int32_t) * 16));
    TRY(grow_slots(h, 16));
    CK(h, cudaStreamSynchronize(h->stream));
    return EGS_OK;
  };
  int rc = boot();
  if (rc != EGS_OK) { fprintf(stderr, "egs_create: %s\n", h->err.c_str()); delete h; return rc; }
  *out = h;
  return EGS_OK;
}

extern "C" int egs_destroy(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  flush_pending(h);
  for (auto &b : h->pin_pool) cudaFreeHost(b.p);
  h->pin_pool.clear();
  rounds_free(&h->rounds);
  void *dev[] = {h->d_core, h->d_mem, h->d_mem_total, h->d_st, h->d_sc, h->d_al, h->d_partials, h->d_ticket, h->d_snap_core, h->d_snap_mem, h->d_snap_total,
                 h->d_result, h->d_ids, h->d_fit, h->d_score, h->d_ev_fit, h->d_ev_score, h->d_ev_gpu, h->d_flush,
                 h->d_o_node, h->d_o_status, h->d_o_fit, h->d_o_alloc, h->d_o_fd, h->d_o_sd, h->d_vec_fit, h->d_vec_score, h->d_ops, h->d_group_off};
  for (void *p : dev) if (p) cudaFree(p);
  if (h->h_result) cudaFreeHost(h->h_result);
  if (h->h_stage) cudaFreeHost(h->h_stage);
  cudaStreamDestroy(h->stream);
  delete h;
  return EGS_OK;
}

extern "C" const char *egs_last_error(egs_handle *h) { return h ? h->err.c_str() : "null handle"; }

extern "C" const char *egs_status_string(int status) {
  switch (status) {
    case EGS_OK: return "";
    case EGS_ERR_NOFIT: return "no enough resource to allocate";                        // gpu.go:126
    case EGS_ERR_NO_OPTION: return "cannot find option of GPU request";                 // node.go:95 (prefix)
    case EGS_ERR_TRANSACT: return "can't trade option";                                 // gpu.go:160 (prefix)
    case EGS_ERR_BAD_ARG: return "bad argument";
    case EGS_ERR_OVERFLOW_GUARD: return "value outside the int32-exact range";
    case EGS_ERR_CUDA: return "cuda error";
    case EGS_ERR_NO_GPU: return "no gpu available on node";                             // node.go:29 (prefix)
    case EGS_ERR_NO_NODE: return "elastic gpu scheduler get node failed";               // scheduler.go:124 (prefix)
    case EGS_ERR_PANIC: return "reference would panic: nil option (node.go:84)";
    case EGS_ERR_COMM: return "nccl error";
  }
  return "unknown";
}

extern "C" uint64_t egs_mix64(uint64_t x) { return mix64(x); }

// NewGPURequest allocate.go:38-53
extern "C" int egs_unit_from_requests(int64_t core, int64_t mem, egs_unit *out) {
  if (!out || core < 0 || mem < 0) return EGS_ERR_BAD_ARG;
  out->core = out->mem = out->count = 0;
  if (core == 0 && mem == 0) { out->core = -1; out->mem = -1; return EGS_OK; }
  if (core >= EGS_CORE_PER_GPU) {
    int64_t k = core / EGS_CORE_PER_GPU;
    out->count = k > 1 << 20 ? 1 << 20 : (int32_t)k;   // anything above EGS_MAX_GPUS never fits
    return EGS_OK;
  }
  if (mem > EGS_MAX_MEM_PER_GPU) return EGS_ERR_OVERFLOW_GUARD;
  out->core = (int32_t)core; out->mem = (int32_t)mem;
  return EGS_OK;
}

// ------------------------------------------------------------------------------- node cache
static int reset_nodes(egs_handle *h, int node0, int n, int full) {
  int ns = (int)h->shapes.size();
  if (ns == 0 || n <= 0) return EGS_OK;
  k_node_reset<<<(n + 255) / 256, 256, 0, h->stream>>>(h->d_st, (size_t)h->n_pad, ns, node0, n, full);
  CK(h, cudaGetLastError());
  return EGS_OK;
}

static int load_rows(egs_handle *h, int node0, int n, int gpu_count, int mem_total, const int32_t *core,
                     const int32_t *mem, bool fresh) {
  if (node0 < 0 || n < 0 || node0 + n > h->max_nodes || gpu_count < 1 || gpu_count > h->g_max) return EGS_ERR_BAD_ARG;
  if (mem_total < 0 || mem_total > EGS_MAX_MEM_PER_GPU) return EGS_ERR_OVERFLOW_GUARD;
  if (n == 0) return EGS_OK;
  const int W = h->row_w;
  size_t cells = (size_t)n * W;
  TRY(ensure_stage(h, cells * 2 * sizeof(int32_t) + (size_t)n * sizeof(int32_t)));
  CK(h, cudaStreamSynchronize(h->stream));   // staging buffer reuse
  int32_t *sc = (int32_t *)h->h_stage, *sm = sc + cells, *st = sm + cells;
  for (int i = 0; i < n; i++) {
    for (int g = 0; g < W; g++) {
      int32_t cv = EGS_PAD, mv = EGS_PAD;
      if (g < gpu_count) {
        cv = core ? core[(size_t)i * gpu_count + g] : EGS_CORE_PER_GPU;
        mv = mem ? mem[(size_t)i * gpu_count + g] : mem_total;
        if (cv < 0 || cv > EGS_MAX_CORE_LOAD || mv < 0 || mv > EGS_MAX_MEM_PER_GPU) return EGS_ERR_OVERFLOW_GUARD;
      }
      sc[(size_t)i * W + g] = cv; sm[(size_t)i * W + g] = mv;
    }
    st[i] = mem_total;
    h->h_gpu_count[node0 + i] = gpu_count; h->h_mem_total[node0 + i] = mem_total;
  }
  CK(h, cudaMemcpyAsync(h->d_core + (size_t)node0 * W, sc, cells * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_mem + (size_t)node0 * W, sm, cells * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_mem_total + node0, st, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  TRY(reset_nodes(h, node0, n, fresh ? 1 : 0));
  if (fresh && node0 == 0 && n >= h->max_nodes) std::fill(h->slot_cold.begin(), h->slot_cold.end(), 1);
  return EGS_OK;
}

// wait for in-flight batches and drop their bookkeeping without applying it
static int discard_pending(egs_handle *h) {
  for (auto &b : h->pending) {
    CK(h, cudaEventSynchronize(b.done));
    pin_put(h, b.buf); cudaEventDestroy(b.done);
  }
  h->pending.clear();
  return EGS_OK;
}

extern "C" int egs_node_set(egs_handle *h, int node_id, int gpu_count, int mem_total_per_gpu) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(flush_pending(h));
  TRY(load_rows(h, node_id, 1, gpu_count, mem_total_per_gpu, nullptr, nullptr, true));
  h->book.drop_nodes(node_id, 1);
  return EGS_OK;
}

extern "C" int egs_node_set_allocatable(egs_handle *h, int node_id, int64_t core_allocatable, int64_t mem_allocatable) {
  if (!h || core_allocatable < 0 || mem_allocatable < 0) return EGS_ERR_BAD_ARG;
  int64_t G = core_allocatable / EGS_CORE_PER_GPU;            // node.go:27
  if (G == 0) return EGS_ERR_NO_GPU;                          // node.go:28-30
  if (G > h->g_max) return EGS_ERR_BAD_ARG;
  int64_t M = mem_allocatable / G;                            // node.go:37-38
  if (M > EGS_MAX_MEM_PER_GPU) return EGS_ERR_OVERFLOW_GUARD;
  return egs_node_set(h, node_id, (int)G, (int)M);
}

extern "C" int egs_state_load(egs_handle *h, int node_id, const int32_t *free_core, const int32_t *free_mem) {
  if (!h || !free_core || !free_mem) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (node_id < 0 || node_id >= h->max_nodes) return EGS_ERR_BAD_ARG;
  if (h->h_gpu_count[node_id] == 0) return EGS_ERR_NO_NODE;
  return load_rows(h, node_id, 1, h->h_gpu_count[node_id], h->h_mem_total[node_id], free_core, free_mem, false);
}

extern "C" int egs_state_load_bulk(egs_handle *h, int node0, int n, int gpu_count, int mem_total,
                                   const int32_t *free_core, const int32_t *free_mem) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  // pending batch results only feed podsMap/podMaps; podMaps (scheduler level) survives a node reload
  TRY(flush_pending(h));
  TRY(load_rows(h, node0, n, gpu_count, mem_total, free_core, free_mem, true));
  h->book.drop_nodes(node0, n);
  return EGS_OK;
}

extern "C" int egs_state_dump(egs_handle *h, int node0, int n, int32_t *free_core, int32_t *free_mem,
                              int32_t *gpu_count, int32_t *mem_total) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (node0 < 0 || n < 0 || node0 + n > h->max_nodes) return EGS_ERR_BAD_ARG;
  size_t cells = (size_t)n * h->row_w;
  TRY(ensure_stage(h, cells * 2 * sizeof(int32_t)));
  int32_t *sc = (int32_t *)h->h_stage, *sm = sc + cells;
  CK(h, cudaMemcpyAsync(sc, h->d_core + (size_t)node0 * h->row_w, cells * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaMemcpyAsync(sm, h->d_mem + (size_t)node0 * h->row_w, cells * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  if (free_core) memcpy(free_core, sc, cells * sizeof(int32_t));
  if (free_mem) memcpy(free_mem, sm, cells * sizeof(int32_t));
  for (int i = 0; i < n; i++) {
    if (gpu_count) gpu_count[i] = h->h_gpu_count[node0 + i];
    if (mem_total) mem_total[i] = h->h_mem_total[node0 + i];
  }
  return EGS_OK;
}

extern "C" int egs_state_snapshot(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  const size_t rows = (size_t)h->n_pad * h->row_w * sizeof(int32_t);
  if (!h->d_snap_core) {
    CK(h, cudaMalloc(&h->d_snap_core, rows));
    CK(h, cudaMalloc(&h->d_snap_mem, rows));
    CK(h, cudaMalloc(&h->d_snap_total, (size_t)h->n_pad * sizeof(int32_t)));
  }
  CK(h, cudaMemcpyAsync(h->d_snap_core, h->d_core, rows, cudaMemcpyDeviceToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_snap_mem, h->d_mem, rows, cudaMemcpyDeviceToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_snap_total, h->d_mem_total, (size_t)h->n_pad * sizeof(int32_t), cudaMemcpyDeviceToDevice, h->stream));
  h->snap_gpu_count = h->h_gpu_count; h->snap_mem_total = h->h_mem_total;
  CK(h, cudaStreamSynchronize(h->stream));
  return EGS_OK;
}

extern "C" int egs_state_restore(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (!h->d_snap_core) return fail(h, EGS_ERR_BAD_ARG, "no snapshot");
  TRY(discard_pending(h));
  const size_t rows = (size_t)h->n_pad * h->row_w * sizeof(int32_t);
  CK(h, cudaMemcpyAsync(h->d_core, h->d_snap_core, rows, cudaMemcpyDeviceToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_mem, h->d_snap_mem, rows, cudaMemcpyDeviceToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_mem_total, h->d_snap_total, (size_t)h->n_pad * sizeof(int32_t), cudaMemcpyDeviceToDevice, h->stream));
  if (!h->shapes.empty())
    CK(h, cudaMemsetAsync(h->d_st, OPT_ABSENT, (size_t)h->n_pad * h->shapes.size(), h->stream));
  std::fill(h->slot_cold.begin(), h->slot_cold.end(), 1);
  h->h_gpu_count = h->snap_gpu_count; h->h_mem_total = h->snap_mem_total;
  h->book.clear();
  return EGS_OK;
}

// ------------------------------------------------------------------------------- verbs
static int ensure_gather(egs_handle *h, size_t n) {
  if (n <= h->gather_cap) return EGS_OK;
  if (h->d_ids) { cudaFree(h->d_ids); cudaFree(h->d_fit); cudaFree(h->d_score); }
  h->d_ids = nullptr; h->gather_cap = 0;
  size_t cap = std::max(n, (size_t)4096);
  CK(h, cudaMalloc(&h->d_ids, cap * sizeof(int32_t)));
  CK(h, cudaMalloc(&h->d_fit, cap));
  CK(h, cudaMalloc(&h->d_score, cap * sizeof(int32_t)));
  h->gather_cap = cap;
  return EGS_OK;
}

static int gather(egs_handle *h, bool score, int n, const int32_t *node_ids, int C, const egs_unit *units,
                  uint8_t *out_fit, int32_t *out_score) {
  if (n < 0 || (n > 0 && !(score ? (void *)out_score : (void *)out_fit))) return EGS_ERR_BAD_ARG;
  int slot;
  TRY(intern(h, C, units, &slot));
  if (n == 0) return EGS_OK;
  h->slot_cold[slot] = 0;
  TRY(ensure_gather(h, (size_t)n));
  TRY(ensure_stage(h, (size_t)n * sizeof(int32_t)));
  GatherArgs a;
  a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total;
  a.n = n; a.n_nodes = h->max_nodes; a.policy = h->policy; a.req = make_req(C, units); a.t = table(h, slot);
  a.ids = nullptr; a.out_fit = h->d_fit; a.out_score = h->d_score; a.panic_flag = h->d_result + 8;
  if (node_ids) {
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(h->h_stage, node_ids, (size_t)n * sizeof(int32_t));
    CK(h, cudaMemcpyAsync(h->d_ids, h->h_stage, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    a.ids = h->d_ids;
  }
  const bool single = is_single(C, units);
  const int grid = (n + 255) / 256;
  if (score) {
    CK(h, cudaMemsetAsync(h->d_result + 8, 0, sizeof(int32_t), h->stream));
    by_width(h, [&](auto W) -> int {
      constexpr int G = decltype(W)::value;
      if (single) k_gather_score<G, true><<<grid, 256, 0, h->stream>>>(a); else k_gather_score<G, false><<<grid, 256, 0, h->stream>>>(a);
      return EGS_OK;
    });
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(h->h_stage, h->d_score, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(h->h_result, h->d_result + 8, sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(out_score, h->h_stage, (size_t)n * sizeof(int32_t));
    return h->h_result[0] ? EGS_ERR_PANIC : EGS_OK;
  }
  by_width(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::value;
    if (single) k_gather_filter<G, true><<<grid, 256, 0, h->stream>>>(a); else k_gather_filter<G, false><<<grid, 256, 0, h->stream>>>(a);
    return EGS_OK;
  });
  CK(h, cudaGetLastError());
  CK(h, cudaMemcpyAsync(h->h_stage, h->d_fit, (size_t)n, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  memcpy(out_fit, h->h_stage, (size_t)n);
  return EGS_OK;
}

extern "C" int egs_filter(egs_handle *h, int n, const int32_t *node_ids, int n_containers, const egs_unit *units,
                          uint8_t *out_fit) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  return gather(h, false, n, node_ids, n_containers, units, out_fit, nullptr);
}
extern "C" int egs_score(egs_handle *h, int n, const int32_t *node_ids, int n_containers, const egs_unit *units,
                         int32_t *out_score) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  return gather(h, true, n, node_ids, n_containers, units, nullptr, out_score);
}

// res[0] had entry, res[1] status, res[2] score; *masks the option's packed masks
static int bind_or_peek(egs_handle *h, int consume, int node_id, int C, const egs_unit *units, uint64_t uid,
                        int32_t *res, uint64_t *masks) {
  if (node_id < 0 || node_id >= h->max_nodes) return EGS_ERR_BAD_ARG;
  if (h->h_gpu_count[node_id] == 0) return EGS_ERR_NO_NODE;
  int slot;
  TRY(intern(h, C, units, &slot));
  TRY(flush_pending(h));
  BindArgs a;
  a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total; a.node = node_id;
  a.req = make_req(C, units); a.t = table(h, slot);
  a.all_st = h->d_st; a.slot_stride = (size_t)h->n_pad; a.n_slots = (int)h->shapes.size();
  const bool known = consume && h->book.in_pods_map(node_id, uid);
  a.skip_transact = known ? 1 : 0; a.consume = consume; a.result = h->d_result;
  by_width(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::value;
    k_bind<G><<<1, 1, 0, h->stream>>>(a);
    return EGS_OK;
  });
  CK(h, cudaGetLastError());
  CK(h, cudaMemcpyAsync(h->h_result, h->d_result, 5 * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  const int32_t *r = h->h_result;
  res[0] = r[0]; res[1] = r[1]; res[2] = r[3];
  *masks = (uint32_t)r[2] | (is_wide(h) ? (uint64_t)(uint32_t)r[4] << 32 : 0);
  if (consume) h->book.record_bind(node_id, uid, res[0] != 0, known, res[1]);
  return EGS_OK;
}

extern "C" int egs_bind(egs_handle *h, int node_id, int n_containers, const egs_unit *units, uint64_t uid,
                        uint8_t *out_alloc_mask) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  int32_t r[3]; uint64_t masks;
  TRY(bind_or_peek(h, 1, node_id, n_containers, units, uid, r, &masks));
  if (out_alloc_mask) put_masks(h, r[1] == EGS_OK ? masks : 0, out_alloc_mask);
  return r[1];
}

extern "C" int egs_option_peek(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                               int32_t *out_valid, int32_t *out_score, uint8_t *out_alloc_mask) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  int32_t r[3]; uint64_t masks;
  TRY(bind_or_peek(h, 0, node_id, n_containers, units, 0, r, &masks));
  if (out_valid) *out_valid = r[0];
  if (out_score) *out_score = r[2];
  if (out_alloc_mask) put_masks(h, r[0] ? masks : 0, out_alloc_mask);
  return EGS_OK;
}

extern "C" int egs_option_dump(egs_handle *h, int n_containers, const egs_unit *units, int node0, int n,
                               uint8_t *out_state, int32_t *out_score, uint8_t *out_alloc_mask) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (node0 < 0 || n < 0 || node0 + n > h->max_nodes) return EGS_ERR_BAD_ARG;
  int slot;
  TRY(intern(h, n_containers, units, &slot));
  if (n == 0) return EGS_OK;
  const OptTable t = table(h, slot);
  const size_t sn = (size_t)n, mb = (size_t)h->mask_b;
  TRY(ensure_stage(h, sn * (1 + 4 + EGS_C * mb)));
  CK(h, cudaStreamSynchronize(h->stream));
  char *s = (char *)h->h_stage;
  int32_t *hs = (int32_t *)s; uint8_t *hst = (uint8_t *)(hs + sn); uint8_t *hal = hst + sn;
  CK(h, cudaMemcpyAsync(hs, t.sc + node0, 4 * sn, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaMemcpyAsync(hst, t.st + node0, sn, cudaMemcpyDeviceToHost, h->stream));
  for (int c = 0; c < EGS_C; c++)
    CK(h, cudaMemcpyAsync(hal + (size_t)c * sn * mb, t.al + ((size_t)c * t.plane + node0) * mb, sn * mb, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < sn; i++) {
    const bool cached = hst[i] == OPT_CACHED;
    if (out_state) out_state[i] = hst[i] == OPT_CACHED ? 1 : hst[i] == OPT_UNFIT ? 2 : 0;
    if (out_score) out_score[i] = cached ? hs[i] : 0;
    if (out_alloc_mask)
      for (int c = 0; c < EGS_C; c++)
        for (size_t b = 0; b < mb; b++)
          out_alloc_mask[(i * EGS_C + c) * mb + b] = (cached && c < n_containers) ? hal[((size_t)c * sn + i) * mb + b] : 0;
  }
  return EGS_OK;
}

static int apply_lists(egs_handle *h, int cancel, int node_id, int C, const egs_unit *units,
                       const int32_t *alloc_off, const int32_t *alloc_idx) {
  return by_width(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::value;
    ApplyArgs<G> a; memset(&a, 0, sizeof a);
    a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total;
    a.op.node = node_id; a.op.cancel = cancel; a.op.req = make_req<ReqW>(C, units);
    a.all_st = h->d_st; a.slot_stride = (size_t)h->n_pad; a.n_slots = (int)h->shapes.size();
    for (int c = 0; c < C; c++) {
      int n = alloc_off ? alloc_off[c + 1] - alloc_off[c] : 0;
      if (n < 0 || n > G || (n > 0 && !alloc_idx)) return EGS_ERR_BAD_ARG;
      a.op.n_idx[c] = n;
      for (int j = 0; j < n; j++) {
        int v = alloc_idx[alloc_off[c] + j];
        if (v < 0 || v >= h->h_gpu_count[node_id]) return EGS_ERR_BAD_ARG;   // the reference would panic
        a.op.idx[c][j] = (int8_t)v;
      }
    }
    k_apply<G><<<1, 1, 0, h->stream>>>(a);
    CK(h, cudaGetLastError());
    return EGS_OK;
  });
}

// AddPod scheduler.go:229-245
extern "C" int egs_pod_apply(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                             const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (node_id < 0 || node_id >= h->max_nodes) return EGS_ERR_BAD_ARG;
  if (h->h_gpu_count[node_id] == 0) return EGS_ERR_NO_NODE;
  TRY(check_units(n_containers, units, EGS_MAX_CONTAINERS_APPLY));
  TRY(flush_pending(h));
  return h->book.account(EGS_MUT_ADD, node_id, uid,
                         [&](int cancel) { return apply_lists(h, cancel, node_id, n_containers, units, alloc_off, alloc_idx); });
}

// NodeAllocator.Add(pod, nil) node.go:148-160 (replay at node load, node.go:52-54)
extern "C" int egs_node_replay_pod(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                                   const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (node_id < 0 || node_id >= h->max_nodes) return EGS_ERR_BAD_ARG;
  if (h->h_gpu_count[node_id] == 0) return EGS_ERR_NO_NODE;
  TRY(check_units(n_containers, units, EGS_MAX_CONTAINERS_APPLY));
  TRY(flush_pending(h));
  return h->book.account(EGS_MUT_REPLAY, node_id, uid,
                         [&](int cancel) { return apply_lists(h, cancel, node_id, n_containers, units, alloc_off, alloc_idx); });
}

// ForgetPod scheduler.go:247-267
extern "C" int egs_pod_cancel(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                              const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(flush_pending(h));
  if (node_id >= 0) {
    if (node_id >= h->max_nodes) return EGS_ERR_BAD_ARG;
    if (h->h_gpu_count[node_id] == 0) return EGS_ERR_NO_NODE;
    TRY(check_units(n_containers, units, EGS_MAX_CONTAINERS_APPLY));
  }
  return h->book.account(EGS_MUT_FORGET, node_id, uid,
                         [&](int cancel) { return apply_lists(h, cancel, node_id, n_containers, units, alloc_off, alloc_idx); });
}

// ------------------------------------------------------------------------------- mutation stream
// caller holds the lock; pending batch bookkeeping already flushed
template <int G> static int mutations_rows(egs_handle *h, int n, const egs_mutation *ops);
static int mutations_apply_locked(egs_handle *h, int n, const egs_mutation *ops) {
  if (n < 0 || (n > 0 && !ops)) return EGS_ERR_BAD_ARG;
  if (n == 0) return EGS_OK;
  // pass 1: validate everything first (a malformed record applies nothing)
  for (int i = 0; i < n; i++) {
    const egs_mutation &m = ops[i];
    if (m.kind < EGS_MUT_ADD || m.kind > EGS_MUT_REPLAY) return EGS_ERR_BAD_ARG;
    if (m.node_id < 0) { if (m.kind != EGS_MUT_FORGET) return EGS_ERR_BAD_ARG; continue; }
    if (m.node_id >= h->max_nodes) return EGS_ERR_BAD_ARG;
    if (h->h_gpu_count[m.node_id] == 0) return EGS_ERR_NO_NODE;
    TRY(check_units(m.n_containers, m.units, EGS_MAX_CONTAINERS_APPLY));
    for (int c = 0; c < m.n_containers; c++) {
      if (m.n_idx[c] < 0 || m.n_idx[c] > EGS_MAX_GPUS) return fail(h, EGS_ERR_BAD_ARG, "a mutation record holds at most EGS_MAX_GPUS indices per container");
      for (int j = 0; j < m.n_idx[c]; j++) if (m.idx[c][j] < 0 || m.idx[c][j] >= h->h_gpu_count[m.node_id]) return EGS_ERR_BAD_ARG;
    }
  }
  return by_width(h, [&](auto W) -> int { return mutations_rows<decltype(W)::value>(h, n, ops); });
}

// passes 2 and 3 of mutations_apply_locked on a handle of row width G
template <int G>
static int mutations_rows(egs_handle *h, int n, const egs_mutation *ops) {
  typedef ApplyOp<G> Op;
  // pass 2: the podsMap / podMaps decisions in record order; the surviving row updates are collected
  std::vector<Op> dev; dev.reserve((size_t)n);
  for (int i = 0; i < n; i++) {
    const egs_mutation &m = ops[i];
    TRY(h->book.account(m.kind, m.node_id, m.uid, [&](int cancel) {
      Op o; memset(&o, 0, sizeof o);
      o.node = m.node_id; o.cancel = cancel; o.req = make_req<ReqW>(m.n_containers, m.units);
      for (int c = 0; c < m.n_containers; c++) { o.n_idx[c] = m.n_idx[c]; for (int j = 0; j < m.n_idx[c]; j++) o.idx[c][j] = m.idx[c][j]; }
      dev.push_back(o);
      return EGS_OK;
    }));
  }
  if (dev.empty()) return EGS_OK;
  // group by node, record order kept inside a node
  std::vector<int> order(dev.size());
  for (size_t i = 0; i < order.size(); i++) order[i] = (int)i;
  std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return dev[x].node < dev[y].node; });
  const size_t nd = dev.size();
  TRY(ensure_stage(h, nd * sizeof(Op) + (nd + 1) * sizeof(int32_t)));
  CK(h, cudaStreamSynchronize(h->stream));
  Op *so = (Op *)h->h_stage; int32_t *sg = (int32_t *)(so + nd);
  int ng = 0;
  for (size_t i = 0; i < nd; i++) {
    so[i] = dev[order[i]];
    if (i == 0 || so[i].node != so[i - 1].node) sg[ng++] = (int32_t)i;
  }
  sg[ng] = (int32_t)nd;
  if (nd > h->ops_cap) {
    if (h->d_ops) { cudaFree(h->d_ops); cudaFree(h->d_group_off); h->d_ops = nullptr; h->d_group_off = nullptr; h->ops_cap = 0; }
    const size_t cap = std::max(nd, (size_t)1024);
    CK(h, cudaMalloc(&h->d_ops, cap * sizeof(Op)));
    CK(h, cudaMalloc(&h->d_group_off, (cap + 1) * sizeof(int32_t)));
    h->ops_cap = cap;
  }
  CK(h, cudaMemcpyAsync(h->d_ops, so, nd * sizeof(Op), cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_group_off, sg, (size_t)(ng + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  ApplyManyArgs<G> ka;
  ka.core = h->d_core; ka.mem = h->d_mem; ka.mem_total = h->d_mem_total; ka.ops = (const Op *)h->d_ops; ka.group_off = h->d_group_off; ka.n_groups = ng;
  ka.all_st = h->d_st; ka.slot_stride = (size_t)h->n_pad; ka.n_slots = (int)h->shapes.size();
  k_apply_many<G><<<(ng + 127) / 128, 128, 0, h->stream>>>(ka);
  CK(h, cudaGetLastError());
  return EGS_OK;
}

extern "C" int egs_mutations_apply(egs_handle *h, int n, const egs_mutation *ops) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(flush_pending(h));
  return mutations_apply_locked(h, n, ops);
}

extern "C" int egs_pod_known(egs_handle *h, uint64_t uid) {
  if (!h) return 0;
  Guard g(h);
  if (flush_pending(h) != EGS_OK) return 0;
  return h->book.in_pod_maps(uid) ? 1 : 0;
}
extern "C" int egs_pod_released(egs_handle *h, uint64_t uid) {
  if (!h) return 0;
  Guard g(h);
  return h->book.released(uid) ? 1 : 0;
}

// ------------------------------------------------------------------------------- batch loop
static int ensure_out(egs_handle *h, int P) {
  if (P <= h->out_cap) return EGS_OK;
  void *old[] = {h->d_o_node, h->d_o_status, h->d_o_fit, h->d_o_alloc, h->d_o_fd, h->d_o_sd};
  for (void *p : old) if (p) cudaFree(p);
  h->out_cap = 0;
  int cap = std::max(P, 1024);
  CK(h, cudaMalloc(&h->d_o_node, sizeof(int32_t) * (size_t)cap));
  CK(h, cudaMalloc(&h->d_o_status, sizeof(int32_t) * (size_t)cap));
  CK(h, cudaMalloc(&h->d_o_fit, sizeof(int32_t) * (size_t)cap));
  CK(h, cudaMalloc(&h->d_o_alloc, (size_t)cap * EGS_C * h->mask_b));
  CK(h, cudaMalloc(&h->d_o_fd, sizeof(unsigned long long) * (size_t)cap));
  CK(h, cudaMalloc(&h->d_o_sd, sizeof(unsigned long long) * (size_t)cap));
  h->out_cap = cap;
  return EGS_OK;
}

// EGS_MODE_RESCAN: one k_pass launch per pod, stream ordered.
static int batch_rescan(egs_handle *h, int P, const int32_t *c_off, const egs_unit *units,
                        const std::vector<int> &slots, PodOut out) {
  const int grid = (h->max_nodes + PASS_THREADS - 1) / PASS_THREADS;
  for (int p = 0; p < P; p++) h->slot_cold[slots[p]] = 0;
  for (int p = 0; p < P; p++) {
    const int C = c_off[p + 1] - c_off[p];
    const egs_unit *u = units + c_off[p];
    PassArgs a;
    a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total; a.core_w = h->d_core; a.mem_w = h->d_mem;
    a.n = h->max_nodes; a.policy = h->policy; a.req = make_req(C, u); a.t = table(h, slots[p]);
    a.all_st = h->d_st; a.slot_stride = (size_t)h->n_pad; a.n_slots = (int)h->shapes.size();
    a.vec_fit = p < h->vec_pods ? h->d_vec_fit + (size_t)p * h->max_nodes : nullptr;
    a.vec_score = p < h->vec_pods ? h->d_vec_score + (size_t)p * h->max_nodes : nullptr;
    a.partials = h->d_partials; a.ticket = h->d_ticket;
    a.pod = p; a.out = out;
    by_width(h, [&](auto W) -> int {
      constexpr int G = decltype(W)::value;
      if (is_single(C, u)) k_pass<G, true><<<grid, PASS_THREADS, 0, h->stream>>>(a);
      else k_pass<G, false><<<grid, PASS_THREADS, 0, h->stream>>>(a);
      return EGS_OK;
    });
    if ((p & 1023) == 0) CK(h, cudaGetLastError());
  }
  CK(h, cudaGetLastError());
  h->k_launches[EGS_K_PASS] += P;
  return EGS_OK;
}

// A wide handle has no rounds engine: EGS_MODE_ROUNDS is refused before the batch touches anything, and
// EGS_MODE_AUTO runs the per-pod engine there.
static int refuse_wide_rounds(egs_handle *h, int mode) {
  return is_wide(h) && mode == EGS_MODE_ROUNDS ? fail(h, EGS_ERR_BAD_ARG, "EGS_MODE_ROUNDS needs g_max <= EGS_MAX_GPUS") : EGS_OK;
}

static int batch_common(egs_handle *h, int mode, int P, const int32_t *c_off, const egs_unit *units,
                        const uint64_t *uids, PodOut out, bool device_out) {
  if (P < 0 || (P > 0 && (!c_off || !units))) return EGS_ERR_BAD_ARG;
  TRY(refuse_wide_rounds(h, mode));
  if (P == 0) return EGS_OK;
  if (h->world > 1 && mode == EGS_MODE_RESCAN) return fail(h, EGS_ERR_BAD_ARG, "EGS_MODE_RESCAN is single-shard");
  std::vector<int> slots((size_t)P);
  for (int p = 0; p < P; p++) {
    const int C = c_off[p + 1] - c_off[p];
    if (C < 1 || C > EGS_C) return EGS_ERR_BAD_ARG;
    TRY(intern(h, C, units + c_off[p], &slots[p]));
  }
  if (uids) {                                    // pods awaiting scheduling must be unknown and distinct
    TRY(flush_pending(h));
    std::unordered_set<uint64_t> seen; seen.reserve((size_t)P * 2);
    for (int p = 0; p < P; p++) {
      if (!seen.insert(uids[p]).second || h->book.in_pod_maps(uids[p])) return fail(h, EGS_ERR_BAD_ARG, "duplicate or known uid");
    }
  }
  PodOut dev = out;
  if (!device_out) {
    TRY(ensure_out(h, P));
    dev.node = h->d_o_node; dev.status = h->d_o_status; dev.fit_count = h->d_o_fit; dev.alloc = h->d_o_alloc;
    dev.fit_digest = h->d_o_fd; dev.score_digest = h->d_o_sd;
  } else {
    TRY(ensure_out(h, P));
    if (!dev.node) dev.node = h->d_o_node;          // uid bookkeeping needs node + status
    if (!dev.status) dev.status = h->d_o_status;
  }
  if (mode == EGS_MODE_AUTO) mode = is_wide(h) ? EGS_MODE_RESCAN : EGS_MODE_ROUNDS;
  int batch_rc = EGS_OK, n_done = P;
  if (mode == EGS_MODE_RESCAN) TRY(batch_rescan(h, P, c_off, units, slots, dev));
  else if (mode == EGS_MODE_ROUNDS) batch_rc = batch_rounds(h, P, c_off, units, slots, dev, &n_done);
  else return EGS_ERR_BAD_ARG;

  // lazy uid bookkeeping: async copy of (node, status), applied on the next uid-dependent verb.  A batch that
  // stopped on an error still records the pods it resolved: their binds are in the rows.
  if (n_done > 0) {
    PendingBatch pb; pb.n = n_done; pb.uid0 = h->next_uid;
    if (uids) pb.uids.assign(uids, uids + n_done); else h->next_uid += (uint64_t)n_done;
    TRY(pin_get(h, 2 * (size_t)n_done, &pb.buf));
    pb.h_node = pb.buf.p; pb.h_status = pb.buf.p + n_done;
    CK(h, cudaMemcpyAsync(pb.h_node, dev.node, sizeof(int32_t) * (size_t)n_done, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(pb.h_status, dev.status, sizeof(int32_t) * (size_t)n_done, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaEventCreateWithFlags(&pb.done, cudaEventDisableTiming));
    CK(h, cudaEventRecord(pb.done, h->stream));
    h->pending.push_back(std::move(pb));
  }
  if (batch_rc != EGS_OK) { cudaStreamSynchronize(h->stream); return batch_rc; }

  if (!device_out) {
    size_t sp = (size_t)P;
    const size_t ab = (size_t)EGS_C * h->mask_b;   // alloc bytes per pod
    TRY(ensure_stage(h, sp * (4 + 4 + 4 + ab + 8 + 8)));
    char *s = (char *)h->h_stage;
    int32_t *hn = (int32_t *)s, *hs = hn + sp, *hf = hs + sp;
    unsigned long long *hfd = (unsigned long long *)(hf + sp), *hsd = hfd + sp;
    uint8_t *ha = (uint8_t *)(hsd + sp);
    if (out.node) CK(h, cudaMemcpyAsync(hn, dev.node, 4 * sp, cudaMemcpyDeviceToHost, h->stream));
    if (out.status) CK(h, cudaMemcpyAsync(hs, dev.status, 4 * sp, cudaMemcpyDeviceToHost, h->stream));
    if (out.fit_count) CK(h, cudaMemcpyAsync(hf, dev.fit_count, 4 * sp, cudaMemcpyDeviceToHost, h->stream));
    if (out.fit_digest) CK(h, cudaMemcpyAsync(hfd, dev.fit_digest, 8 * sp, cudaMemcpyDeviceToHost, h->stream));
    if (out.score_digest) CK(h, cudaMemcpyAsync(hsd, dev.score_digest, 8 * sp, cudaMemcpyDeviceToHost, h->stream));
    if (out.alloc) CK(h, cudaMemcpyAsync(ha, dev.alloc, ab * sp, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    if (out.node) memcpy(out.node, hn, 4 * sp);
    if (out.status) memcpy(out.status, hs, 4 * sp);
    if (out.fit_count) memcpy(out.fit_count, hf, 4 * sp);
    if (out.fit_digest) memcpy(out.fit_digest, hfd, 8 * sp);
    if (out.score_digest) memcpy(out.score_digest, hsd, 8 * sp);
    if (out.alloc) memcpy(out.alloc, ha, ab * sp);
  } else {
    CK(h, cudaStreamSynchronize(h->stream));
  }
  return EGS_OK;
}

extern "C" int egs_schedule_batch(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                                  const uint64_t *uids, int32_t *out_node, int32_t *out_status,
                                  uint8_t *out_alloc_mask, int32_t *out_fit_count, uint64_t *out_fit_digest,
                                  uint64_t *out_score_digest) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  PodOut o; o.node = out_node; o.status = out_status; o.alloc = out_alloc_mask; o.fit_count = out_fit_count;
  o.fit_digest = (unsigned long long *)out_fit_digest; o.score_digest = (unsigned long long *)out_score_digest;
  return batch_common(h, mode, n_pods, c_off, units, uids, o, false);
}

extern "C" int egs_schedule_batch_mut(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                                      const uint64_t *uids, int n_mut, const int32_t *mut_at, const egs_mutation *muts,
                                      int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                                      int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest) {
  if (!h || n_pods < 0 || n_mut < 0 || (n_mut > 0 && (!mut_at || !muts)) || (n_pods > 0 && (!c_off || !units))) return EGS_ERR_BAD_ARG;
  for (int j = 0; j < n_mut; j++)
    if (mut_at[j] < 0 || mut_at[j] > n_pods || (j > 0 && mut_at[j] < mut_at[j - 1])) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(refuse_wide_rounds(h, mode));                              // before the first record is applied
  // segments of pods between mutation points; the lock is held throughout, exactly one "call at a time"
  int p = 0, j = 0;
  while (p < n_pods || j < n_mut) {
    int j1 = j;
    while (j1 < n_mut && mut_at[j1] == p) j1++;
    if (j1 > j) {
      TRY(flush_pending(h));
      TRY(mutations_apply_locked(h, j1 - j, muts + j));
      j = j1;
    }
    if (p >= n_pods) break;
    const int q = j < n_mut ? mut_at[j] : n_pods;                // next mutation point (> p)
    PodOut o;
    o.node = out_node ? out_node + p : nullptr; o.status = out_status ? out_status + p : nullptr;
    o.alloc = out_alloc_mask ? out_alloc_mask + (size_t)p * EGS_C * h->mask_b : nullptr; o.fit_count = out_fit_count ? out_fit_count + p : nullptr;
    o.fit_digest = out_fit_digest ? (unsigned long long *)out_fit_digest + p : nullptr;
    o.score_digest = out_score_digest ? (unsigned long long *)out_score_digest + p : nullptr;
    // the segment's pods as a batch of its own: offsets rebased
    std::vector<int32_t> off((size_t)(q - p) + 1);
    for (int i = p; i <= q; i++) off[(size_t)(i - p)] = c_off[i] - c_off[p];
    TRY(batch_common(h, mode, q - p, off.data(), units + c_off[p], uids ? uids + p : nullptr, o, false));
    p = q;
  }
  return EGS_OK;
}

extern "C" int egs_schedule_batch_vec(egs_handle *h, int n_pods, const int32_t *c_off, const egs_unit *units,
                                      const uint64_t *uids, int vec_pods, uint8_t *out_vec_fit, int32_t *out_vec_score,
                                      int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                                      int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest) {
  if (!h || vec_pods < 0 || (vec_pods > 0 && (!out_vec_fit || !out_vec_score))) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (h->world > 1) return fail(h, EGS_ERR_BAD_ARG, "egs_schedule_batch_vec is single-shard");
  vec_pods = std::min(vec_pods, n_pods);
  const size_t cells = (size_t)vec_pods * h->max_nodes;
  if (cells > h->vec_cap) {
    if (h->d_vec_fit) { cudaFree(h->d_vec_fit); cudaFree(h->d_vec_score); h->d_vec_fit = nullptr; h->d_vec_score = nullptr; h->vec_cap = 0; }
    CK(h, cudaMalloc(&h->d_vec_fit, cells));
    CK(h, cudaMalloc(&h->d_vec_score, cells * sizeof(int32_t)));
    h->vec_cap = cells;
  }
  PodOut o; o.node = out_node; o.status = out_status; o.alloc = out_alloc_mask; o.fit_count = out_fit_count;
  o.fit_digest = (unsigned long long *)out_fit_digest; o.score_digest = (unsigned long long *)out_score_digest;
  h->vec_pods = vec_pods;
  const int rc = batch_common(h, EGS_MODE_RESCAN, n_pods, c_off, units, uids, o, false);
  h->vec_pods = 0;
  if (rc != EGS_OK) return rc;
  if (cells) {
    CK(h, cudaMemcpy(out_vec_fit, h->d_vec_fit, cells, cudaMemcpyDeviceToHost));
    CK(h, cudaMemcpy(out_vec_score, h->d_vec_score, cells * sizeof(int32_t), cudaMemcpyDeviceToHost));
  }
  return EGS_OK;
}

extern "C" int egs_schedule_batch_device(egs_handle *h, int mode, int n_pods, const int32_t *h_c_off,
                                         const egs_unit *h_units, int32_t *d_out_node, int32_t *d_out_status,
                                         uint8_t *d_out_alloc_mask, int32_t *d_out_fit_count,
                                         uint64_t *d_out_fit_digest, uint64_t *d_out_score_digest) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if ((uintptr_t)d_out_alloc_mask % ((uintptr_t)EGS_C * h->mask_b))     // one packed word per pod (write_pod_out)
    return fail(h, EGS_ERR_BAD_ARG, "d_out_alloc_mask must be aligned to EGS_MAX_CONTAINERS * EGS_MASK_BYTES(g_max)");
  PodOut o; o.node = d_out_node; o.status = d_out_status; o.alloc = d_out_alloc_mask; o.fit_count = d_out_fit_count;
  o.fit_digest = (unsigned long long *)d_out_fit_digest; o.score_digest = (unsigned long long *)d_out_score_digest;
  return batch_common(h, mode, n_pods, h_c_off, h_units, nullptr, o, true);
}

// ------------------------------------------------------------------------------- sharding
extern "C" int egs_shard_range(int max_nodes, int rank, int world, int *lo, int *hi) {
  if (max_nodes < 1 || world < 1 || rank < 0 || rank >= world || !lo || !hi) return EGS_ERR_BAD_ARG;
  // contiguous node ranges, boundaries on multiples of 128 (k_select reads 4-node vectors)
  auto cut = [&](int r) { return r >= world ? max_nodes : (int)((int64_t)max_nodes * r / world) / 128 * 128; };
  *lo = cut(rank); *hi = cut(rank + 1);
  return EGS_OK;
}

extern "C" int egs_shard_set(egs_handle *h, int rank, int world) {
  if (!h || world < 1 || world > RD || rank < 0 || rank >= world) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (is_wide(h)) return fail(h, EGS_ERR_BAD_ARG, "the sharded engine is the rounds engine: it needs g_max <= EGS_MAX_GPUS");
  h->rank = rank; h->world = world;
  egs_shard_range(h->max_nodes, rank, world, &h->lo, &h->hi);
  return EGS_OK;
}
extern "C" int egs_comm_unique_id(uint8_t out_id[128]) { return rounds_comm_unique_id(out_id); }
extern "C" int egs_comm_init_local(egs_handle **handles, int world) { return rounds_comm_init_local(handles, world); }
extern "C" int egs_comm_init(egs_handle *h, const uint8_t id[128]) {
  if (!h || !id) return EGS_ERR_BAD_ARG;
  Guard g(h);
  return rounds_comm_init(h, id);
}

// ------------------------------------------------------------------------------- instrumentation
extern "C" int egs_profile_evaluate(egs_handle *h, int n_containers, const egs_unit *units, int iters,
                                    int flush_l2, float *out_ms_per_launch) {
  if (!h || iters < 1 || !out_ms_per_launch) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(check_units(n_containers, units));
  const size_t np = (size_t)h->n_pad;
  if (!h->d_ev_fit) {
    CK(h, cudaMalloc(&h->d_ev_fit, np));
    CK(h, cudaMalloc(&h->d_ev_score, np * sizeof(int32_t)));
    CK(h, cudaMalloc(&h->d_ev_gpu, np * EGS_C * h->mask_b));
  }
  const size_t flush_bytes = (size_t)256 << 20;
  if (flush_l2 && !h->d_flush) CK(h, cudaMalloc(&h->d_flush, flush_bytes));
  EvalArgs a;
  a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total; a.lo = 0; a.n = h->max_nodes; a.policy = h->policy;
  a.req = make_req(n_containers, units); a.fit = h->d_ev_fit; a.score = h->d_ev_score; a.gpu = h->d_ev_gpu; a.plane = np;
  a.v_fit = 1; a.v_unfit = 0;
  const bool single = is_single(n_containers, units);
  int items = 2;                                  // nodes per thread (tuning knob for experiments)
  if (const char *ev = getenv("EGS_EVAL_ITEMS")) items = atoi(ev);
  if (items != 1 && items != 2 && items != 4) items = 2;
  if (is_wide(h)) items = 1;                      // a 16-wide row already keeps 8 loads of 16 B in flight per thread
  const int grid = (h->max_nodes + 256 * items - 1) / (256 * items);
  auto launch = [&]() {
    by_width(h, [&](auto W) -> int {
      constexpr int G = decltype(W)::value;
      if (!single) k_evaluate<G, false, 1><<<(h->max_nodes + 255) / 256, 256, 0, h->stream>>>(a);
      else if constexpr (G == EGS_G) {
        if (items == 1) k_evaluate<G, true, 1><<<grid, 256, 0, h->stream>>>(a);
        else if (items == 2) k_evaluate<G, true, 2><<<grid, 256, 0, h->stream>>>(a);
        else k_evaluate<G, true, 4><<<grid, 256, 0, h->stream>>>(a);
      } else {
        k_evaluate<G, true, 1><<<grid, 256, 0, h->stream>>>(a);
      }
      return EGS_OK;
    });
  };
  cudaEvent_t e0, e1;
  CK(h, cudaEventCreate(&e0)); CK(h, cudaEventCreate(&e1));
  double total = 0;
  for (int it = 0; it < iters; it++) {
    if (flush_l2) CK(h, cudaMemsetAsync(h->d_flush, it & 0xff, flush_bytes, h->stream));
    CK(h, cudaEventRecord(e0, h->stream));
    launch();
    CK(h, cudaEventRecord(e1, h->stream));
    CK(h, cudaEventSynchronize(e1));
    float ms = 0;
    CK(h, cudaEventElapsedTime(&ms, e0, e1));
    total += ms;
  }
  CK(h, cudaGetLastError());
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  h->k_launches[EGS_K_EVALUATE] += iters; h->k_ms[EGS_K_EVALUATE] += total;
  *out_ms_per_launch = (float)(total / iters);
  return EGS_OK;
}

extern "C" int egs_rounds_stats(egs_handle *h, int64_t out[8]) {
  if (!h || !out) return EGS_ERR_BAD_ARG;
  Guard g(h);
  const RoundsState &R = h->rounds;
  out[0] = R.rounds; out[1] = R.pods; out[2] = R.tracked;
  for (int i = 0; i < 4; i++) out[3 + i] = R.stops[i];
  out[7] = 0;
  return EGS_OK;
}

// debug: cycle counters of k_resolve sections (only filled when built with -DEGS_RESOLVE_PROF)
extern "C" int egs_debug_resolve_prof(egs_handle *h, long long out[RPROF]) {
  if (!h || !out) return EGS_ERR_BAD_ARG;
  Guard g(h);
  memcpy(out, h->rounds.prof, sizeof(long long) * RPROF);
  return EGS_OK;
}

extern "C" int egs_get_stream(egs_handle *h, void **out_stream) {
  if (!h || !out_stream) return EGS_ERR_BAD_ARG;
  *out_stream = (void *)h->stream;
  return EGS_OK;
}

extern "C" int egs_profile_get(egs_handle *h, int kernel_id, int64_t *out_launches, double *out_ms) {
  if (!h || kernel_id < 0 || kernel_id >= EGS_K_COUNT) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (out_launches) *out_launches = h->k_launches[kernel_id];
  if (out_ms) *out_ms = h->k_ms[kernel_id];
  return EGS_OK;
}
extern "C" int egs_profile_reset(egs_handle *h, int enable_timing) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  memset(h->k_launches, 0, sizeof h->k_launches);
  for (double &d : h->k_ms) d = 0;
  h->timing = enable_timing;
  return EGS_OK;
}
#include "egs_rounds_impl.cuh"
