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

#include "buffers.h"
#include "egs_kernels.cuh"
#include "egs_rounds.cuh"
#include "pod_book.h"

struct Shape { int C; egs_unit u[EGS_CA]; };

// Pinned host buffer holding (node[n], status[n]) of a batch.  Recycled through egs_handle::pin_pool: allocating and
// freeing pinned memory cost milliseconds and synchronise the device -- too much for a small batch on the extender's path.
using PinBuf = PinnedBuf<int32_t>;
struct PendingBatch {           // results of a batch whose uid bookkeeping is applied lazily
  int n; uint64_t uid0; std::vector<uint64_t> uids; int32_t *h_node, *h_status; PinBuf buf; cudaEvent_t done;
};

struct ShapeCacheEnt { uint64_t h; int slot; };   // open-addressing entry of egs_handle::shape_cache

// The rows of every node: free_core / free_mem / mem_total on the device and the host's gpu_count / mem_total, which
// also say which nodes are set.  A snapshot and a checkpoint each hold one; its device buffers are allocated on the
// first save.
struct RowImage {
  DeviceBuf<int32_t> d_core, d_mem, d_mem_total;
  std::vector<int32_t> h_gpu_count, h_mem_total;
  int save(egs_handle *h);
  int load(egs_handle *h) const;
};

// The option tables of `slots` slots: state, score and masks, each array one contiguous slice per slot (table()).  The
// handle's live tables and a checkpoint's copy.
struct OptTables {
  DeviceBuf<uint8_t> st; DeviceBuf<int32_t> sc; DeviceBuf<uint8_t> al;
  int slots = 0;
  int grow(egs_handle *h, int cap);                      // keeps every slot held; the new slots' states read OPT_ABSENT
  int copy_from(egs_handle *h, const OptTables &o, int n);   // slots [0, n) of o
};

// egs_checkpoint_save: the complete scheduler state but the PodBook, which keeps its own undo journal.  The device
// buffers are allocated on the first save and grown when more shapes are interned.
struct Checkpoint {
  bool open = false;
  RowImage rows;
  OptTables tables;
  int n_shapes = 0;                       // shapes interned at the save; later ones are forgotten by the rollback
  std::vector<char> slot_cold;
  std::vector<ShapeCacheEnt> shape_cache;
  uint64_t next_uid = 0;
};

struct egs_handle {
  int policy = 0, max_nodes = 0, n_pad = 0, g_max = 0, device = 0, n_sm = 0;
  int row_w = EGS_G, mask_b = 1;          // EGS_ROW_WIDTH(g_max), EGS_MASK_BYTES(g_max)
  int c_max = EGS_C, planes = EGS_C;      // largest pod Traded, EGS_MASKS_PER_POD(c_max)
  int rank = 0, world = 1, lo = 0, hi = 0;
  cudaStream_t stream = nullptr;
  DeviceBuf<int32_t> d_core, d_mem, d_mem_total;
  std::vector<int32_t> h_gpu_count, h_mem_total;
  RowImage snap;
  OptTables tables;
  std::vector<Shape> shapes;
  std::vector<char> slot_cold;            // option table of the slot holds only OPT_ABSENT (nothing evaluated yet)
  std::unordered_map<std::string, int> shape_ids;
  using ShapeCacheEnt = ::ShapeCacheEnt;
  std::vector<ShapeCacheEnt> shape_cache = std::vector<ShapeCacheEnt>(1024, ShapeCacheEnt{0, -1});   // open addressing
  // reference bookkeeping that never reaches the device
  PodBook book;                                                 // podsMap / podMaps / releasedPodMap
  std::vector<PendingBatch> pending;                            // batches whose results have not reached the book
  std::vector<PinBuf> pin_pool;                                 // idle pinned result buffers (at most PIN_POOL_MAX)
  uint64_t next_uid = 0x8000000000000000ull;
  // scratch
  DeviceBuf<Partial> d_partials; DeviceBuf<unsigned int> d_ticket; DeviceBuf<int32_t> d_result;
  PinnedBuf<int32_t> h_result;
  DeviceBuf<int32_t> d_ids; DeviceBuf<uint8_t> d_fit; DeviceBuf<int32_t> d_score;
  DeviceBuf<int32_t> d_miss; DeviceBuf<unsigned long long> d_keys; int leaf_grid = 0;   // leaf-split Trade (sidecar)
  PinnedBuf<char> h_stage;                                      // staging
  // eval scratch (profile)
  DeviceBuf<uint8_t> d_ev_fit; DeviceBuf<int32_t> d_ev_score; DeviceBuf<uint8_t> d_ev_gpu; DeviceBuf<char> d_flush;
  // batch outputs
  DeviceBuf<int32_t> d_o_node, d_o_status, d_o_fit; DeviceBuf<uint8_t> d_o_alloc;
  DeviceBuf<unsigned long long> d_o_fd, d_o_sd;
  DeviceBuf<char> d_ops; DeviceBuf<int32_t> d_group_off;       // egs_mutations_apply: ApplyOp<row_w>[]
  DeviceBuf<uint8_t> d_vec_fit; DeviceBuf<int32_t> d_vec_score;              // egs_schedule_batch_vec
  DeviceBuf<uint64_t> d_set;                                    // egs_schedule_batch_nodes: the running run's node set
  DeviceBuf<int32_t> d_hr; DeviceBuf<unsigned long long> d_hr_sum;   // egs_headroom: count | failed, summaries
  // profiling
  int64_t k_launches[EGS_K_COUNT] = {0}; double k_ms[EGS_K_COUNT] = {0}; int timing = 0;
  RoundsState rounds;
  Checkpoint ck;
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

// The one place the handle's geometry picks a kernel instantiation: f(Geo<G, NP>()) with G the row width and NP the
// mask planes per pod -- (8, 4), (16, 4) on a wide handle, or (8, 8) on a sidecar handle.
template <int G_, int NP_> struct Geo { static constexpr int G = G_, NP = NP_; };
template <class F>
static int by_geometry(const egs_handle *h, F &&f) {
  if (h->row_w == 16) return f(Geo<16, EGS_C>());
  return h->planes == EGS_CA ? f(Geo<EGS_G, EGS_CA>()) : f(Geo<EGS_G, EGS_C>());
}
static bool is_wide(const egs_handle *h) { return h->row_w > EGS_G; }
static bool is_sidecar(const egs_handle *h) { return h->planes > EGS_C; }

// Packed option masks (container c at bits [G*c, G*c + G)) -> EGS_MASKS_PER_POD little-endian masks of mask_b bytes.
static void put_masks(const egs_handle *h, uint64_t masks, uint8_t *out) {
  for (int c = 0; c < h->planes; c++)
    for (int b = 0; b < h->mask_b; b++) out[c * h->mask_b + b] = (uint8_t)(masks >> (h->row_w * c + 8 * b));
}

static int ensure_stage(egs_handle *h, size_t bytes) {
  if (bytes > h->h_stage.cap()) CK(h, grow(h->stream, false, to(h->h_stage, std::max(bytes, (size_t)1 << 20))));
  return EGS_OK;
}

static OptTable table(egs_handle *h, int slot) {
  OptTable t;
  t.plane = (size_t)h->n_pad;
  t.st = h->tables.st + (size_t)slot * h->n_pad;
  t.sc = h->tables.sc + (size_t)slot * h->n_pad;
  t.al = h->tables.al + (size_t)slot * h->planes * h->n_pad * h->mask_b;
  return t;
}

int OptTables::grow(egs_handle *h, int cap) {
  const size_t np = (size_t)h->n_pad, al_plane = np * h->planes * h->mask_b;
  CK(h, ::grow(h->stream, true, to(st, np * cap), to(sc, np * cap), to(al, al_plane * cap)));
  CK(h, cudaMemsetAsync(st + np * slots, OPT_ABSENT, np * (cap - slots), h->stream));
  slots = cap;
  return EGS_OK;
}

int OptTables::copy_from(egs_handle *h, const OptTables &o, int n) {
  const size_t np = (size_t)h->n_pad, al_plane = np * h->planes * h->mask_b;
  CK(h, st.copy_from(o.st, np * n, h->stream));
  CK(h, sc.copy_from(o.sc, np * n, h->stream));
  CK(h, al.copy_from(o.al, al_plane * n, h->stream));
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
  if (C >= 1 && C <= h->c_max && u) {
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

static std::string shape_key(int C, const egs_unit *u) {
  std::string key((const char *)&C, sizeof C);
  key.append((const char *)u, sizeof(egs_unit) * C);
  return key;
}

static int intern_slow(egs_handle *h, int C, const egs_unit *u, int *slot) {
  TRY(check_units(C, u, h->c_max));
  const std::string key = shape_key(C, u);
  auto it = h->shape_ids.find(key);
  if (it != h->shape_ids.end()) { *slot = it->second; return EGS_OK; }
  int s = (int)h->shapes.size();
  if (s + 1 > h->tables.slots) TRY(h->tables.grow(h, std::max(s + 1, h->tables.slots * 2)));
  Shape sh; sh.C = C; memset(sh.u, 0, sizeof sh.u); memcpy(sh.u, u, sizeof(egs_unit) * C);
  h->shapes.push_back(sh);
  h->slot_cold.push_back(1);
  h->shape_ids.emplace(key, s);
  *slot = s;
  return EGS_OK;
}

static bool is_single(int C, const egs_unit *u) { return C == 1 && u[0].count == 0 && u[0].core >= 0 && u[0].mem >= 0; }

// Digit width of the leaf space on this handle: every node has at most g_max GPUs (trade_leaf_space).
static int leaf_bits(const egs_handle *h) { return h->g_max <= 1 ? 0 : h->g_max <= 2 ? 1 : h->g_max <= 4 ? 2 : 3; }
static int n_branch(int C, const egs_unit *u) {
  int n = 0;
  for (int i = 0; i < C; i++) n += u[i].count == 0 ? 1 : 0;
  return n;
}
// Shapes whose leaf space has more than 2^LEAF_SPLIT_LOG2 leaves are Traded by the leaf-split kernels; smaller ones
// by the one-thread DFS inside k_pass / k_gather_*.  2^12 = 8^4 is the DFS's worst case on a handle without sidecars.
constexpr int LEAF_SPLIT_LOG2 = 12;
static bool leaf_split(const egs_handle *h, int C, const egs_unit *u) {
  return is_sidecar(h) && leaf_bits(h) * n_branch(C, u) > LEAF_SPLIT_LOG2;
}

// The leaf-split Trade of every candidate of slot `slot` whose option is absent (k_trade_probe, k_trade_leaves,
// k_trade_commit; egs_kernels.cuh), enqueued on the stream.  d_ids == nullptr: nodes [0, n).  With d_score the probe is
// also Score's read of the cache and the commit raises d_panic.  With d_set only the nodes of that set are Traded.
static int trade_misses(egs_handle *h, int slot, int C, const egs_unit *u, const int32_t *d_ids, int n,
                        int32_t *d_score, int *d_panic, const uint64_t *d_set = nullptr) {
  if (n <= 0) return EGS_OK;
  if ((size_t)n > h->d_miss.cap()) {
    const size_t cap = std::max((size_t)n, (size_t)h->n_pad);
    CK(h, grow(h->stream, false, to(h->d_miss, cap), to(h->d_keys, cap)));
  }
  if (!h->leaf_grid) {
    int per_sm = 0;
    CK(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_trade_leaves, LEAF_THREADS, 0));
    h->leaf_grid = std::max(per_sm, 1) * h->n_sm;
  }
  unsigned int *d_n = reinterpret_cast<unsigned int *>(h->d_ticket.get()) + 1;   // ticket[0] belongs to k_pass
  CK(h, cudaMemsetAsync(d_n, 0, sizeof(unsigned int), h->stream));
  const OptTable t = table(h, slot);
  ProbeArgs pa;
  pa.st = t.st; pa.sc = t.sc; pa.ids = d_ids; pa.n = n; pa.n_nodes = h->max_nodes;
  pa.miss = h->d_miss; pa.n_miss = d_n; pa.keys = h->d_keys; pa.out_score = d_score;
  const int grid = (n + 255) / 256;
  if (d_set) k_trade_probe_nodes<<<grid, 256, 0, h->stream>>>(pa, NodeSet{d_set});
  else k_trade_probe<<<grid, 256, 0, h->stream>>>(pa);
  LeafArgs la;
  la.core = h->d_core; la.mem = h->d_mem; la.mem_total = h->d_mem_total;
  la.policy = h->policy; la.bits = leaf_bits(h); la.nbranch = n_branch(C, u);
  const int nleaf = 1 << (la.bits * la.nbranch);
  la.tiles = (nleaf + LEAF_THREADS * LEAF_CHUNK - 1) / (LEAF_THREADS * LEAF_CHUNK);
  la.req = make_req<ReqW>(C, u);
  la.miss = h->d_miss; la.n_miss = d_n; la.keys = h->d_keys;
  k_trade_leaves<<<h->leaf_grid, LEAF_THREADS, 0, h->stream>>>(la);
  k_trade_commit<<<grid, 256, 0, h->stream>>>(la, t, d_panic);
  CK(h, cudaGetLastError());
  return EGS_OK;
}

constexpr size_t PIN_POOL_MAX = 4;
static void pin_put(egs_handle *h, PinBuf b) {
  if (b && h->pin_pool.size() < PIN_POOL_MAX) h->pin_pool.push_back(std::move(b));
}

// Waits for the batches in flight and moves their results into the book (apply), or drops them.
static int settle_pending(egs_handle *h, bool apply) {
  for (auto &b : h->pending) {
    CK(h, cudaEventSynchronize(b.done));
    if (apply && b.uids.empty()) h->book.add_run(b.uid0, b.n, b.h_node, b.h_status);     // library-assigned uids
    else if (apply) h->book.add_batch(b.uids.data(), b.n, b.h_node, b.h_status);
    pin_put(h, std::move(b.buf)); cudaEventDestroy(b.done);
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
    if (h->pin_pool[i].cap() >= n && (best < 0 || h->pin_pool[i].cap() < h->pin_pool[(size_t)best].cap())) best = (int)i;
  if (best >= 0) { *out = std::move(h->pin_pool[(size_t)best]); h->pin_pool.erase(h->pin_pool.begin() + best); return EGS_OK; }
  CK(h, grow(h->stream, false, to(*out, std::max(n, (size_t)4096))));
  return EGS_OK;
}

static void checkpoint_free(egs_handle *h) {
  if (h->ck.rows.d_core) cudaStreamSynchronize(h->stream);   // no copy into the checkpoint's buffers is still in flight
  h->ck = Checkpoint();
  h->book.drop_checkpoint();
}

// The handle and everything it owns; the stream goes last.
static void free_handle(egs_handle *h) {
  cudaStream_t s = h->stream;
  delete h;
  if (s) cudaStreamDestroy(s);
}

// ------------------------------------------------------------------------------- lifecycle
extern "C" int egs_create(int policy, int max_nodes, int g_max, int device, egs_handle **out) {
  return egs_create_ex(policy, max_nodes, g_max, EGS_MAX_CONTAINERS, device, out);
}

extern "C" int egs_create_ex(int policy, int max_nodes, int g_max, int c_max, int device, egs_handle **out) {
  if (!out || max_nodes < 1 || g_max < 1 || g_max > EGS_MAX_GPUS_WIDE || (policy != EGS_BINPACK && policy != EGS_SPREAD))
    return EGS_ERR_BAD_ARG;
  if (c_max < 1 || c_max > EGS_MAX_CONTAINERS_APPLY) return EGS_ERR_BAD_ARG;
  if (c_max > EGS_MAX_CONTAINERS && g_max > EGS_MAX_GPUS) return EGS_ERR_BAD_ARG;   // 128-bit masks, 2^32 leaves
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1 || device < 0 || device >= ndev) return EGS_ERR_CUDA;
  egs_handle *h = new egs_handle();
  h->policy = policy; h->max_nodes = max_nodes; h->g_max = g_max; h->device = device;
  h->row_w = EGS_ROW_WIDTH(g_max); h->mask_b = EGS_MASK_BYTES(g_max);
  h->c_max = std::max(c_max, EGS_MAX_CONTAINERS); h->planes = EGS_MASKS_PER_POD(c_max);
  h->n_pad = (max_nodes + 1023) / 1024 * 1024;
  h->lo = 0; h->hi = max_nodes;
  h->h_gpu_count.assign(max_nodes, 0); h->h_mem_total.assign(max_nodes, 0);
  auto boot = [&]() -> int {
    CK(h, cudaSetDevice(device));
    CK(h, cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
    CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    const size_t cells = (size_t)h->n_pad * h->row_w;
    CK(h, grow(h->stream, false, to(h->d_core, cells), to(h->d_mem, cells), to(h->d_mem_total, h->n_pad)));
    CK(h, cudaMemsetAsync(h->d_mem_total, 0, (size_t)h->n_pad * sizeof(int32_t), h->stream));
    // EGS_PAD == 0x80000000: fill through a pinned pattern-free path (memset is per byte)
    std::vector<int32_t> pad(cells, EGS_PAD);
    CK(h, cudaMemcpy(h->d_core, pad.data(), cells * sizeof(int32_t), cudaMemcpyHostToDevice));
    CK(h, cudaMemcpy(h->d_mem, pad.data(), cells * sizeof(int32_t), cudaMemcpyHostToDevice));
    int nblk = (h->n_pad + PASS_THREADS - 1) / PASS_THREADS;
    CK(h, grow(h->stream, false, to(h->d_partials, nblk), to(h->d_ticket, 4), to(h->d_result, 16), to(h->h_result, 16)));
    CK(h, cudaMemsetAsync(h->d_ticket, 0, sizeof(unsigned int) * 4, h->stream));
    TRY(h->tables.grow(h, 16));
    CK(h, cudaStreamSynchronize(h->stream));
    return EGS_OK;
  };
  int rc = boot();
  if (rc != EGS_OK) { fprintf(stderr, "egs_create: %s\n", h->err.c_str()); free_handle(h); return rc; }
  *out = h;
  return EGS_OK;
}

extern "C" int egs_destroy(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  settle_pending(h, true);
  rounds_free(&h->rounds);
  free_handle(h);
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
static int check_node(const egs_handle *h, int node) {
  if (node < 0 || node >= h->max_nodes) return EGS_ERR_BAD_ARG;
  return h->h_gpu_count[node] == 0 ? EGS_ERR_NO_NODE : EGS_OK;
}

static int reset_nodes(egs_handle *h, int node0, int n, int full) {
  int ns = (int)h->shapes.size();
  if (ns == 0 || n <= 0) return EGS_OK;
  k_node_reset<<<(n + 255) / 256, 256, 0, h->stream>>>(h->tables.st, (size_t)h->n_pad, ns, node0, n, full);
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
  int32_t *sc = (int32_t *)h->h_stage.get(), *sm = sc + cells, *st = sm + cells;
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

extern "C" int egs_node_set(egs_handle *h, int node_id, int gpu_count, int mem_total_per_gpu) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(settle_pending(h, true));
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
  TRY(check_node(h, node_id));
  return load_rows(h, node_id, 1, h->h_gpu_count[node_id], h->h_mem_total[node_id], free_core, free_mem, false);
}

extern "C" int egs_state_load_bulk(egs_handle *h, int node0, int n, int gpu_count, int mem_total,
                                   const int32_t *free_core, const int32_t *free_mem) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  // pending batch results only feed podsMap/podMaps; podMaps (scheduler level) survives a node reload
  TRY(settle_pending(h, true));
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
  int32_t *sc = (int32_t *)h->h_stage.get(), *sm = sc + cells;
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

int RowImage::save(egs_handle *h) {
  const size_t cells = (size_t)h->n_pad * h->row_w;
  if (!d_core) CK(h, grow(h->stream, false, to(d_core, cells), to(d_mem, cells), to(d_mem_total, h->n_pad)));
  CK(h, d_core.copy_from(h->d_core, cells, h->stream));
  CK(h, d_mem.copy_from(h->d_mem, cells, h->stream));
  CK(h, d_mem_total.copy_from(h->d_mem_total, h->n_pad, h->stream));
  h_gpu_count = h->h_gpu_count; h_mem_total = h->h_mem_total;
  return EGS_OK;
}

int RowImage::load(egs_handle *h) const {
  const size_t cells = (size_t)h->n_pad * h->row_w;
  CK(h, h->d_core.copy_from(d_core, cells, h->stream));
  CK(h, h->d_mem.copy_from(d_mem, cells, h->stream));
  CK(h, h->d_mem_total.copy_from(d_mem_total, h->n_pad, h->stream));
  h->h_gpu_count = h_gpu_count; h->h_mem_total = h_mem_total;
  return EGS_OK;
}

extern "C" int egs_state_snapshot(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(h->snap.save(h));
  CK(h, cudaStreamSynchronize(h->stream));
  return EGS_OK;
}

extern "C" int egs_state_restore(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (!h->snap.d_core) return fail(h, EGS_ERR_BAD_ARG, "no snapshot");
  TRY(settle_pending(h, false));
  TRY(h->snap.load(h));
  if (!h->shapes.empty())
    CK(h, cudaMemsetAsync(h->tables.st, OPT_ABSENT, (size_t)h->n_pad * h->shapes.size(), h->stream));
  std::fill(h->slot_cold.begin(), h->slot_cold.end(), 1);
  h->book.clear();
  return EGS_OK;
}

extern "C" int egs_checkpoint_save(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(settle_pending(h, true));                   // batches still pending belong to the saved state
  Checkpoint &k = h->ck;
  k.open = false;                                 // an earlier checkpoint is overwritten from here on
  h->book.drop_checkpoint();
  const int ns = (int)h->shapes.size();
  if (ns > k.tables.slots) TRY(k.tables.grow(h, std::max(ns, h->tables.slots)));
  TRY(k.rows.save(h));
  TRY(k.tables.copy_from(h, h->tables, ns));
  k.n_shapes = ns;
  k.slot_cold = h->slot_cold;
  k.shape_cache = h->shape_cache;
  k.next_uid = h->next_uid;
  h->book.checkpoint();
  k.open = true;
  return EGS_OK;
}

extern "C" int egs_checkpoint_rollback(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  Checkpoint &k = h->ck;
  if (!k.open) return fail(h, EGS_ERR_BAD_ARG, "no checkpoint: egs_checkpoint_save first");
  TRY(settle_pending(h, false));                  // batches after the save whose results never reached the book
  const int ns = (int)h->shapes.size();
  TRY(k.rows.load(h));
  TRY(h->tables.copy_from(h, k.tables, k.n_shapes));   // the tables may have been reallocated since: slot offsets hold
  if (ns > k.n_shapes)                            // slots interned since the save read OPT_ABSENT again
    CK(h, cudaMemsetAsync(h->tables.st + (size_t)k.n_shapes * h->n_pad, OPT_ABSENT, (size_t)(ns - k.n_shapes) * h->n_pad, h->stream));
  for (int s = k.n_shapes; s < ns; s++) h->shape_ids.erase(shape_key(h->shapes[s].C, h->shapes[s].u));
  h->shapes.resize((size_t)k.n_shapes);
  h->slot_cold = k.slot_cold;
  h->shape_cache = k.shape_cache;
  h->next_uid = k.next_uid;
  h->book.rollback();
  return EGS_OK;
}

extern "C" int egs_checkpoint_drop(egs_handle *h) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  checkpoint_free(h);
  return EGS_OK;
}

// ------------------------------------------------------------------------------- verbs
static int gather(egs_handle *h, bool score, int n, const int32_t *node_ids, int C, const egs_unit *units,
                  uint8_t *out_fit, int32_t *out_score) {
  if (n < 0 || (n > 0 && !(score ? (void *)out_score : (void *)out_fit))) return EGS_ERR_BAD_ARG;
  int slot;
  TRY(intern(h, C, units, &slot));
  if (n == 0) return EGS_OK;
  h->slot_cold[slot] = 0;
  if ((size_t)n > h->d_ids.cap()) {
    const size_t cap = std::max((size_t)n, (size_t)4096);
    CK(h, grow(h->stream, false, to(h->d_ids, cap), to(h->d_fit, cap), to(h->d_score, cap)));
  }
  TRY(ensure_stage(h, (size_t)n * sizeof(int32_t)));
  const int32_t *d_ids = nullptr;
  if (node_ids) {
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(h->h_stage, node_ids, (size_t)n * sizeof(int32_t));
    CK(h, cudaMemcpyAsync(h->d_ids, h->h_stage, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    d_ids = h->d_ids;
  }
  const bool single = is_single(C, units), split = leaf_split(h, C, units);
  const int grid = (n + 255) / 256;
  // the arguments in the geometry's request type
  auto args = [&](auto W) {
    GatherArgsT<ReqOf<decltype(W)::NP>> a;
    a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total;
    a.n = n; a.n_nodes = h->max_nodes; a.policy = h->policy; a.req = make_req<ReqOf<decltype(W)::NP>>(C, units);
    a.t = table(h, slot); a.ids = d_ids; a.out_fit = h->d_fit; a.out_score = h->d_score; a.panic_flag = h->d_result + 8;
    return a;
  };
  if (score) {
    CK(h, cudaMemsetAsync(h->d_result + 8, 0, sizeof(int32_t), h->stream));
    if (split) {                                   // the probe is Score's read; the commit raises the panic flag
      TRY(trade_misses(h, slot, C, units, d_ids, n, h->d_score, h->d_result + 8));
    } else {
      by_geometry(h, [&](auto W) -> int {
        constexpr int G = decltype(W)::G, NP = decltype(W)::NP;
        if (single) k_gather_score<G, NP, true><<<grid, 256, 0, h->stream>>>(args(W));
        else k_gather_score<G, NP, false><<<grid, 256, 0, h->stream>>>(args(W));
        return EGS_OK;
      });
    }
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(h->h_stage, h->d_score, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(h->h_result, h->d_result + 8, sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(out_score, h->h_stage, (size_t)n * sizeof(int32_t));
    return h->h_result[0] ? EGS_ERR_PANIC : EGS_OK;
  }
  if (split) TRY(trade_misses(h, slot, C, units, d_ids, n, nullptr, nullptr));   // k_gather_filter then only reads
  by_geometry(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::G, NP = decltype(W)::NP;
    if (single) k_gather_filter<G, NP, true><<<grid, 256, 0, h->stream>>>(args(W));
    else k_gather_filter<G, NP, false><<<grid, 256, 0, h->stream>>>(args(W));
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
  TRY(check_node(h, node_id));
  int slot;
  TRY(intern(h, C, units, &slot));
  TRY(settle_pending(h, true));
  const bool known = consume && h->book.in_pods_map(node_id, uid);
  by_geometry(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::G, NP = decltype(W)::NP;
    BindArgsT<ReqOf<NP>> a;
    a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total; a.node = node_id;
    a.req = make_req<ReqOf<NP>>(C, units); a.t = table(h, slot);
    a.all_st = h->tables.st; a.slot_stride = (size_t)h->n_pad; a.n_slots = (int)h->shapes.size();
    a.skip_transact = known ? 1 : 0; a.consume = consume; a.result = h->d_result;
    k_bind<G, NP><<<1, 1, 0, h->stream>>>(a);
    return EGS_OK;
  });
  CK(h, cudaGetLastError());
  CK(h, cudaMemcpyAsync(h->h_result, h->d_result, 5 * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  const int32_t *r = h->h_result;
  res[0] = r[0]; res[1] = r[1]; res[2] = r[3];
  *masks = (uint32_t)r[2] | (h->row_w * h->planes > 32 ? (uint64_t)(uint32_t)r[4] << 32 : 0);   // a 64-bit packed word
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
  const int np = h->planes;
  TRY(ensure_stage(h, sn * (1 + 4 + np * mb)));
  CK(h, cudaStreamSynchronize(h->stream));
  char *s = h->h_stage.get();
  int32_t *hs = (int32_t *)s; uint8_t *hst = (uint8_t *)(hs + sn); uint8_t *hal = hst + sn;
  CK(h, cudaMemcpyAsync(hs, t.sc + node0, 4 * sn, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaMemcpyAsync(hst, t.st + node0, sn, cudaMemcpyDeviceToHost, h->stream));
  for (int c = 0; c < np; c++)
    CK(h, cudaMemcpyAsync(hal + (size_t)c * sn * mb, t.al + ((size_t)c * t.plane + node0) * mb, sn * mb, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < sn; i++) {
    const bool cached = hst[i] == OPT_CACHED;
    if (out_state) out_state[i] = hst[i] == OPT_CACHED ? 1 : hst[i] == OPT_UNFIT ? 2 : 0;
    if (out_score) out_score[i] = cached ? hs[i] : 0;
    if (out_alloc_mask)
      for (int c = 0; c < np; c++)
        for (size_t b = 0; b < mb; b++)
          out_alloc_mask[(i * np + c) * mb + b] = (cached && c < n_containers) ? hal[((size_t)c * sn + i) * mb + b] : 0;
  }
  return EGS_OK;
}

static int apply_lists(egs_handle *h, int cancel, int node_id, int C, const egs_unit *units,
                       const int32_t *alloc_off, const int32_t *alloc_idx) {
  return by_geometry(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::G;
    ApplyArgs<G> a; memset(&a, 0, sizeof a);
    a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total;
    a.op.node = node_id; a.op.cancel = cancel; a.op.req = make_req<ReqW>(C, units);
    a.all_st = h->tables.st; a.slot_stride = (size_t)h->n_pad; a.n_slots = (int)h->shapes.size();
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
  TRY(check_node(h, node_id));
  TRY(check_units(n_containers, units, EGS_MAX_CONTAINERS_APPLY));
  TRY(settle_pending(h, true));
  return h->book.account(EGS_MUT_ADD, node_id, uid,
                         [&](int cancel) { return apply_lists(h, cancel, node_id, n_containers, units, alloc_off, alloc_idx); });
}

// NodeAllocator.Add(pod, nil) node.go:148-160 (replay at node load, node.go:52-54)
extern "C" int egs_node_replay_pod(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                                   const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(check_node(h, node_id));
  TRY(check_units(n_containers, units, EGS_MAX_CONTAINERS_APPLY));
  TRY(settle_pending(h, true));
  return h->book.account(EGS_MUT_REPLAY, node_id, uid,
                         [&](int cancel) { return apply_lists(h, cancel, node_id, n_containers, units, alloc_off, alloc_idx); });
}

// ForgetPod scheduler.go:247-267
extern "C" int egs_pod_cancel(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                              const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(settle_pending(h, true));
  if (node_id >= 0) {
    TRY(check_node(h, node_id));
    TRY(check_units(n_containers, units, EGS_MAX_CONTAINERS_APPLY));
  }
  return h->book.account(EGS_MUT_FORGET, node_id, uid,
                         [&](int cancel) { return apply_lists(h, cancel, node_id, n_containers, units, alloc_off, alloc_idx); });
}

// ------------------------------------------------------------------------------- mutation stream
// caller holds the lock; pending batch bookkeeping already flushed
template <int G> static int mutations_rows(egs_handle *h, int n, const egs_mutation *ops);
// A record of a set node (node_id >= 0): its node, units and index lists.
static int check_record(egs_handle *h, const egs_mutation &m) {
  TRY(check_node(h, m.node_id));
  TRY(check_units(m.n_containers, m.units, EGS_MAX_CONTAINERS_APPLY));
  for (int c = 0; c < m.n_containers; c++) {
    if (m.n_idx[c] < 0 || m.n_idx[c] > EGS_MAX_GPUS) return fail(h, EGS_ERR_BAD_ARG, "a mutation record holds at most EGS_MAX_GPUS indices per container");
    for (int j = 0; j < m.n_idx[c]; j++) if (m.idx[c][j] < 0 || m.idx[c][j] >= h->h_gpu_count[m.node_id]) return EGS_ERR_BAD_ARG;
  }
  return EGS_OK;
}
static int mutations_apply_locked(egs_handle *h, int n, const egs_mutation *ops) {
  if (n < 0 || (n > 0 && !ops)) return EGS_ERR_BAD_ARG;
  if (n == 0) return EGS_OK;
  // pass 1: validate everything first (a malformed record applies nothing)
  for (int i = 0; i < n; i++) {
    const egs_mutation &m = ops[i];
    if (m.kind < EGS_MUT_ADD || m.kind > EGS_MUT_REPLAY) return EGS_ERR_BAD_ARG;
    if (m.node_id < 0) { if (m.kind != EGS_MUT_FORGET) return EGS_ERR_BAD_ARG; continue; }
    TRY(check_record(h, m));
  }
  return by_geometry(h, [&](auto W) -> int { return mutations_rows<decltype(W)::G>(h, n, ops); });
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
      dev.push_back(apply_op_of<G>(m, cancel));
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
  Op *so = (Op *)h->h_stage.get(); int32_t *sg = (int32_t *)(so + nd);
  int ng = 0;
  for (size_t i = 0; i < nd; i++) {
    so[i] = dev[order[i]];
    if (i == 0 || so[i].node != so[i - 1].node) sg[ng++] = (int32_t)i;
  }
  sg[ng] = (int32_t)nd;
  if (nd * sizeof(Op) > h->d_ops.cap()) {
    const size_t cap = std::max(nd, (size_t)1024);
    CK(h, grow(h->stream, false, to(h->d_ops, cap * sizeof(Op)), to(h->d_group_off, cap + 1)));
  }
  CK(h, cudaMemcpyAsync(h->d_ops, so, nd * sizeof(Op), cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaMemcpyAsync(h->d_group_off, sg, (size_t)(ng + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  ApplyManyArgs<G> ka;
  ka.core = h->d_core; ka.mem = h->d_mem; ka.mem_total = h->d_mem_total; ka.ops = (const Op *)h->d_ops.get(); ka.group_off = h->d_group_off; ka.n_groups = ng;
  ka.all_st = h->tables.st; ka.slot_stride = (size_t)h->n_pad; ka.n_slots = (int)h->shapes.size();
  k_apply_many<G><<<(ng + 127) / 128, 128, 0, h->stream>>>(ka);
  CK(h, cudaGetLastError());
  return EGS_OK;
}

extern "C" int egs_mutations_apply(egs_handle *h, int n, const egs_mutation *ops) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(settle_pending(h, true));
  return mutations_apply_locked(h, n, ops);
}

extern "C" int egs_pod_known(egs_handle *h, uint64_t uid) {
  if (!h) return 0;
  Guard g(h);
  if (settle_pending(h, true) != EGS_OK) return 0;
  return h->book.in_pod_maps(uid) ? 1 : 0;
}
extern "C" int egs_pod_released(egs_handle *h, uint64_t uid) {
  if (!h) return 0;
  Guard g(h);
  return h->book.released(uid) ? 1 : 0;
}

// ------------------------------------------------------------------------------- batch loop
// The caller's outputs of one batch call: the six per-pod arrays, device pointers when `device` and host pointers
// otherwise, each of which may be null; and egs_schedule_batch_vec's full fit / score vectors, [vec_pods][max_nodes]
// on the device, read only for pods below vec_pods.
struct BatchOut {
  PodOut pod; bool device;
  uint8_t *vec_fit = nullptr; int32_t *vec_score = nullptr; int vec_pods = 0;
  BatchOut(int32_t *node, int32_t *status, uint8_t *alloc, int32_t *fit_count, uint64_t *fit_digest,
           uint64_t *score_digest, bool device)
      : pod{node, status, fit_count, alloc, (unsigned long long *)fit_digest, (unsigned long long *)score_digest},
        device(device) {}
};

// The outputs of pods [p, ...) of a batch whose outputs are `o`: every pointer advanced by p pods.
static BatchOut out_from(const egs_handle *h, BatchOut o, int p) {
  auto at = [p](auto *&a, size_t per_pod) { if (a) a += (size_t)p * per_pod; };
  at(o.pod.node, 1); at(o.pod.status, 1); at(o.pod.fit_count, 1); at(o.pod.fit_digest, 1); at(o.pod.score_digest, 1);
  at(o.pod.alloc, (size_t)h->planes * h->mask_b);
  o.vec_pods = std::max(o.vec_pods - p, 0);
  if (o.vec_pods) { at(o.vec_fit, h->max_nodes); at(o.vec_score, h->max_nodes); }
  return o;
}

static int ensure_out(egs_handle *h, int P) {
  if ((size_t)P <= h->d_o_node.cap()) return EGS_OK;
  const size_t cap = (size_t)std::max(P, 1024);
  CK(h, grow(h->stream, false, to(h->d_o_node, cap), to(h->d_o_status, cap), to(h->d_o_fit, cap),
             to(h->d_o_alloc, cap * h->planes * h->mask_b), to(h->d_o_fd, cap), to(h->d_o_sd, cap)));
  return EGS_OK;
}

// EGS_MODE_RESCAN: one k_pass launch per pod into the device outputs `out`, stream ordered; k_pass_nodes under d_set.
static int batch_rescan(egs_handle *h, int P, const int32_t *c_off, const egs_unit *units,
                        const std::vector<int> &slots, const BatchOut &out, const uint64_t *d_set) {
  const int grid = (h->max_nodes + PASS_THREADS - 1) / PASS_THREADS;
  for (int p = 0; p < P; p++) h->slot_cold[slots[p]] = 0;
  for (int p = 0; p < P; p++) {
    const int C = c_off[p + 1] - c_off[p];
    const egs_unit *u = units + c_off[p];
    // a shape past the one-thread DFS is Traded on every node without an option first: k_pass then only reads caches
    if (leaf_split(h, C, u)) TRY(trade_misses(h, slots[p], C, u, nullptr, h->max_nodes, nullptr, nullptr, d_set));
    by_geometry(h, [&](auto W) -> int {
      constexpr int G = decltype(W)::G, NP = decltype(W)::NP;
      PassArgsT<ReqOf<NP>> a;
      a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total; a.core_w = h->d_core; a.mem_w = h->d_mem;
      a.n = h->max_nodes; a.policy = h->policy; a.req = make_req<ReqOf<NP>>(C, u); a.t = table(h, slots[p]);
      a.all_st = h->tables.st; a.slot_stride = (size_t)h->n_pad; a.n_slots = (int)h->shapes.size();
      a.vec_fit = p < out.vec_pods ? out.vec_fit + (size_t)p * h->max_nodes : nullptr;
      a.vec_score = p < out.vec_pods ? out.vec_score + (size_t)p * h->max_nodes : nullptr;
      a.partials = h->d_partials; a.ticket = h->d_ticket;
      a.pod = p; a.out = out.pod;
      if (d_set && is_single(C, u)) k_pass_nodes<G, NP, true><<<grid, PASS_THREADS, 0, h->stream>>>(a, NodeSet{d_set});
      else if (d_set) k_pass_nodes<G, NP, false><<<grid, PASS_THREADS, 0, h->stream>>>(a, NodeSet{d_set});
      else if (is_single(C, u)) k_pass<G, NP, true><<<grid, PASS_THREADS, 0, h->stream>>>(a);
      else k_pass<G, NP, false><<<grid, PASS_THREADS, 0, h->stream>>>(a);
      return EGS_OK;
    });
    if ((p & 1023) == 0) CK(h, cudaGetLastError());
  }
  CK(h, cudaGetLastError());
  h->k_launches[EGS_K_PASS] += P;
  return EGS_OK;
}

// Wide and sidecar handles have no rounds engine: EGS_MODE_AUTO runs the per-pod engine there.
static bool per_pod_only(const egs_handle *h) { return is_wide(h) || is_sidecar(h); }

// The argument checks every batch entry point makes, under the lock, before it applies or allocates anything.
static int check_batch(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units) {
  if (n_pods < 0 || (n_pods > 0 && (!c_off || !units))) return EGS_ERR_BAD_ARG;
  if (mode == EGS_MODE_ROUNDS && is_wide(h)) return fail(h, EGS_ERR_BAD_ARG, "EGS_MODE_ROUNDS needs g_max <= EGS_MAX_GPUS");
  if (mode == EGS_MODE_ROUNDS && is_sidecar(h)) return fail(h, EGS_ERR_BAD_ARG, "EGS_MODE_ROUNDS needs c_max <= EGS_MAX_CONTAINERS");
  return EGS_OK;
}

// Pods [0, P) of one segment, P > 0.  c_off[p] is the offset of pod p's units from `units`; out: the segment's
// outputs.  d_set: the pods' node set on the device (egs_schedule_batch_nodes), nullptr for every node.
static int batch_common(egs_handle *h, int mode, int P, const int32_t *c_off, const egs_unit *units,
                        const uint64_t *uids, const BatchOut &out, const uint64_t *d_set) {
  if (h->world > 1 && mode == EGS_MODE_RESCAN) return fail(h, EGS_ERR_BAD_ARG, "EGS_MODE_RESCAN is single-shard");
  std::vector<int> slots((size_t)P);
  for (int p = 0; p < P; p++) {
    const int C = c_off[p + 1] - c_off[p];
    if (C < 1 || C > h->c_max) return EGS_ERR_BAD_ARG;
    TRY(intern(h, C, units + c_off[p], &slots[p]));
  }
  if (uids) {                                    // pods awaiting scheduling must be unknown and distinct
    TRY(settle_pending(h, true));
    std::unordered_set<uint64_t> seen; seen.reserve((size_t)P * 2);
    for (int p = 0; p < P; p++) {
      if (!seen.insert(uids[p]).second || h->book.in_pod_maps(uids[p])) return fail(h, EGS_ERR_BAD_ARG, "duplicate or known uid");
    }
  }
  TRY(ensure_out(h, P));
  BatchOut dev = out;                            // the kernels' outputs: the handle's buffers stand in for host ones
  if (!out.device) dev.pod = PodOut{h->d_o_node, h->d_o_status, h->d_o_fit, h->d_o_alloc, h->d_o_fd, h->d_o_sd};
  if (!dev.pod.node) dev.pod.node = h->d_o_node;          // uid bookkeeping needs node + status
  if (!dev.pod.status) dev.pod.status = h->d_o_status;
  if (mode == EGS_MODE_AUTO) mode = per_pod_only(h) ? EGS_MODE_RESCAN : EGS_MODE_ROUNDS;
  int batch_rc = EGS_OK, n_done = P;
  if (mode == EGS_MODE_RESCAN) TRY(batch_rescan(h, P, c_off, units, slots, dev, d_set));
  else if (mode == EGS_MODE_ROUNDS) batch_rc = batch_rounds(h, P, slots, dev.pod, &n_done, d_set);
  else return EGS_ERR_BAD_ARG;

  // lazy uid bookkeeping: async copy of (node, status), applied on the next uid-dependent verb.  A batch that
  // stopped on an error still records the pods it resolved: their binds are in the rows.
  if (n_done > 0) {
    PendingBatch pb; pb.n = n_done; pb.uid0 = h->next_uid;
    if (uids) pb.uids.assign(uids, uids + n_done); else h->next_uid += (uint64_t)n_done;
    TRY(pin_get(h, 2 * (size_t)n_done, &pb.buf));
    pb.h_node = pb.buf; pb.h_status = pb.buf + n_done;
    CK(h, cudaMemcpyAsync(pb.h_node, dev.pod.node, sizeof(int32_t) * (size_t)n_done, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(pb.h_status, dev.pod.status, sizeof(int32_t) * (size_t)n_done, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaEventCreateWithFlags(&pb.done, cudaEventDisableTiming));
    CK(h, cudaEventRecord(pb.done, h->stream));
    h->pending.push_back(std::move(pb));
  }
  if (batch_rc != EGS_OK) { cudaStreamSynchronize(h->stream); return batch_rc; }

  if (out.device) { CK(h, cudaStreamSynchronize(h->stream)); return EGS_OK; }

  // host outputs: each requested array is staged through pinned memory
  const PodOut &o = out.pod, &d = dev.pod;
  const size_t sp = (size_t)P, ab = (size_t)h->planes * h->mask_b;   // alloc bytes per pod
  const struct { void *to; const void *from; size_t bytes; } arrays[] = {
      {o.node, d.node, 4 * sp}, {o.status, d.status, 4 * sp}, {o.fit_count, d.fit_count, 4 * sp},
      {o.fit_digest, d.fit_digest, 8 * sp}, {o.score_digest, d.score_digest, 8 * sp}, {o.alloc, d.alloc, ab * sp}};
  TRY(ensure_stage(h, sp * (4 + 4 + 4 + 8 + 8 + ab)));
  char *s = h->h_stage.get();
  for (const auto &x : arrays) {
    if (x.to) CK(h, cudaMemcpyAsync(s, x.from, x.bytes, cudaMemcpyDeviceToHost, h->stream));
    s += x.bytes;
  }
  CK(h, cudaStreamSynchronize(h->stream));
  s = h->h_stage.get();
  for (const auto &x : arrays) {
    if (x.to) memcpy(x.to, s, x.bytes);
    s += x.bytes;
  }
  return EGS_OK;
}

// The one driver of the batch entry points.  Pods [0, n_pods) run in segments, each one batch_common call: the
// mutation records due at pod p (mut_at) are applied, then pods [p, q) run, q being the next mutation point or,
// under node sets, the first pod of another set.  A set is uploaded when its run starts.  Without records or sets
// the batch is one segment.  The lock is held throughout, exactly one "call at a time"; an error stops the loop and
// keeps what earlier segments applied.
struct NodeSets { const uint64_t *sets = nullptr; const int32_t *pod_set = nullptr; };
static int run_segments(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                        const uint64_t *uids, const BatchOut &out, int n_mut = 0, const int32_t *mut_at = nullptr,
                        const egs_mutation *muts = nullptr, const NodeSets &ns = NodeSets()) {
  const size_t words = EGS_NODE_SET_WORDS((size_t)h->max_nodes);
  auto set_of = [&](int p) { return ns.pod_set ? ns.pod_set[p] : 0; };
  if (ns.sets && words > h->d_set.cap()) CK(h, grow(h->stream, false, to(h->d_set, words)));
  int p = 0, j = 0, loaded = -1;
  while (p < n_pods || j < n_mut) {
    int j1 = j;
    while (j1 < n_mut && mut_at[j1] == p) j1++;
    if (j1 > j) {
      TRY(settle_pending(h, true));
      TRY(mutations_apply_locked(h, j1 - j, muts + j));
      j = j1;
    }
    if (p >= n_pods) break;
    int q = j < n_mut ? mut_at[j] : n_pods;                      // next mutation point (> p)
    if (ns.sets) {
      for (int i = p + 1; i < q; i++) if (set_of(i) != set_of(p)) { q = i; break; }
      if (set_of(p) != loaded) {
        loaded = set_of(p);
        CK(h, cudaMemcpyAsync(h->d_set, ns.sets + (size_t)loaded * words, words * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
      }
    }
    TRY(batch_common(h, mode, q - p, c_off + p, units, uids ? uids + p : nullptr, out_from(h, out, p),
                     ns.sets ? h->d_set.get() : nullptr));
    p = q;
  }
  return EGS_OK;
}

extern "C" int egs_schedule_batch(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                                  const uint64_t *uids, int32_t *out_node, int32_t *out_status,
                                  uint8_t *out_alloc_mask, int32_t *out_fit_count, uint64_t *out_fit_digest,
                                  uint64_t *out_score_digest) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(check_batch(h, mode, n_pods, c_off, units));
  const BatchOut o(out_node, out_status, out_alloc_mask, out_fit_count, out_fit_digest, out_score_digest, false);
  return run_segments(h, mode, n_pods, c_off, units, uids, o);
}

extern "C" int egs_schedule_batch_mut(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                                      const uint64_t *uids, int n_mut, const int32_t *mut_at, const egs_mutation *muts,
                                      int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                                      int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest) {
  if (!h || n_mut < 0 || (n_mut > 0 && (!mut_at || !muts))) return EGS_ERR_BAD_ARG;
  for (int j = 0; j < n_mut; j++)
    if (mut_at[j] < 0 || mut_at[j] > n_pods || (j > 0 && mut_at[j] < mut_at[j - 1])) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(check_batch(h, mode, n_pods, c_off, units));               // before the first record is applied
  const BatchOut o(out_node, out_status, out_alloc_mask, out_fit_count, out_fit_digest, out_score_digest, false);
  return run_segments(h, mode, n_pods, c_off, units, uids, o, n_mut, mut_at, muts);
}

extern "C" int egs_schedule_batch_nodes(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                                        const uint64_t *uids, int n_sets, const uint64_t *sets, const int32_t *pod_set,
                                        int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                                        int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest) {
  if (!h || n_sets < 1 || !sets) return EGS_ERR_BAD_ARG;
  if (pod_set)
    for (int p = 0; p < n_pods; p++) if (pod_set[p] < 0 || pod_set[p] >= n_sets) return EGS_ERR_BAD_ARG;
  const size_t words = EGS_NODE_SET_WORDS((size_t)h->max_nodes);
  if (h->max_nodes % 64) {                                       // no bit at or beyond max_nodes
    const uint64_t beyond = ~0ull << (h->max_nodes % 64);
    for (int s = 0; s < n_sets; s++) if (sets[(size_t)s * words + words - 1] & beyond) return EGS_ERR_BAD_ARG;
  }
  Guard g(h);
  TRY(check_batch(h, mode, n_pods, c_off, units));
  NodeSets ns; ns.sets = sets; ns.pod_set = pod_set;
  const BatchOut o(out_node, out_status, out_alloc_mask, out_fit_count, out_fit_digest, out_score_digest, false);
  return run_segments(h, mode, n_pods, c_off, units, uids, o, 0, nullptr, nullptr, ns);
}

extern "C" int egs_schedule_batch_vec(egs_handle *h, int n_pods, const int32_t *c_off, const egs_unit *units,
                                      const uint64_t *uids, int vec_pods, uint8_t *out_vec_fit, int32_t *out_vec_score,
                                      int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                                      int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest) {
  if (!h || vec_pods < 0 || (vec_pods > 0 && (!out_vec_fit || !out_vec_score))) return EGS_ERR_BAD_ARG;
  Guard g(h);
  TRY(check_batch(h, EGS_MODE_RESCAN, n_pods, c_off, units));
  if (h->world > 1) return fail(h, EGS_ERR_BAD_ARG, "egs_schedule_batch_vec is single-shard");
  BatchOut o(out_node, out_status, out_alloc_mask, out_fit_count, out_fit_digest, out_score_digest, false);
  o.vec_pods = std::min(vec_pods, n_pods);
  const size_t cells = (size_t)o.vec_pods * h->max_nodes;
  if (cells > h->d_vec_fit.cap()) CK(h, grow(h->stream, false, to(h->d_vec_fit, cells), to(h->d_vec_score, cells)));
  o.vec_fit = h->d_vec_fit; o.vec_score = h->d_vec_score;
  TRY(run_segments(h, EGS_MODE_RESCAN, n_pods, c_off, units, uids, o));
  if (cells) {
    CK(h, cudaMemcpyAsync(out_vec_fit, h->d_vec_fit, cells, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(out_vec_score, h->d_vec_score, cells * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
  }
  return EGS_OK;
}

extern "C" int egs_schedule_batch_device(egs_handle *h, int mode, int n_pods, const int32_t *h_c_off,
                                         const egs_unit *h_units, int32_t *d_out_node, int32_t *d_out_status,
                                         uint8_t *d_out_alloc_mask, int32_t *d_out_fit_count,
                                         uint64_t *d_out_fit_digest, uint64_t *d_out_score_digest) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if ((uintptr_t)d_out_alloc_mask % ((uintptr_t)h->planes * h->mask_b))     // one packed word per pod (write_pod_out)
    return fail(h, EGS_ERR_BAD_ARG, "d_out_alloc_mask must be aligned to EGS_MASKS_PER_POD(c_max) * EGS_MASK_BYTES(g_max)");
  TRY(check_batch(h, mode, n_pods, h_c_off, h_units));
  const BatchOut o(d_out_node, d_out_status, d_out_alloc_mask, d_out_fit_count, d_out_fit_digest, d_out_score_digest, true);
  return run_segments(h, mode, n_pods, h_c_off, h_units, nullptr, o);
}

// ------------------------------------------------------------------------------- capacity
// Every argument is checked before a shape is interned or anything is launched.  One k_headroom launch per shape,
// all on the stream after whatever batch is still in flight, and one synchronisation for the copies back.
extern "C" int egs_headroom(egs_handle *h, int n_shapes, const int32_t *c_off, const egs_unit *units, int node0, int n,
                            const uint64_t *set, int32_t limit, int32_t *out_count, int32_t *out_failed,
                            int64_t *out_summary) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (n_shapes < 1 || !c_off || !units) return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: n_shapes >= 1 shapes in c_off / units");
  if (!out_count && !out_failed && !out_summary) return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: no output");
  if (limit < 1 || limit > EGS_HEADROOM_MAX_LIMIT) return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: limit outside [1, EGS_HEADROOM_MAX_LIMIT]");
  if (node0 < 0 || n < 0 || node0 > h->max_nodes - n) return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: node range outside [0, max_nodes)");
  if (h->world > 1 && (node0 < h->lo || node0 + n > h->hi))
    return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: on a sharded handle the range must lie inside the rank's egs_shard_range");
  const size_t words = EGS_NODE_SET_WORDS((size_t)h->max_nodes);
  if (set && h->max_nodes % 64 && (set[words - 1] & (~0ull << (h->max_nodes % 64))))
    return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: node set bit at or beyond max_nodes");
  for (int s = 0; s < n_shapes; s++) {
    const int C = c_off[s + 1] - c_off[s];
    if (c_off[s] < 0 || C < 1 || C > h->c_max) return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: shape with 0 or more than c_max containers");
    const int rc = check_units(C, units + c_off[s], h->c_max);
    if (rc != EGS_OK) return fail(h, rc, "egs_headroom: malformed unit");
    if (leaf_split(h, C, units + c_off[s]))
      return fail(h, EGS_ERR_BAD_ARG, "egs_headroom: shapes Traded by the leaf-split kernels (more than 2^12 leaves) are not served");
  }
  std::vector<int> slots((size_t)n_shapes);
  for (int s = 0; s < n_shapes; s++) TRY(intern(h, c_off[s + 1] - c_off[s], units + c_off[s], &slots[s]));
  const size_t cells = (size_t)n_shapes * n;
  if (2 * cells > h->d_hr.cap()) CK(h, grow(h->stream, false, to(h->d_hr, std::max(2 * cells, (size_t)h->n_pad))));
  if ((size_t)n_shapes * 4 > h->d_hr_sum.cap()) CK(h, grow(h->stream, false, to(h->d_hr_sum, (size_t)n_shapes * 4)));
  CK(h, cudaMemsetAsync(h->d_hr_sum, 0, (size_t)n_shapes * 4 * sizeof(unsigned long long), h->stream));
  if (set) {
    if (words > h->d_set.cap()) CK(h, grow(h->stream, false, to(h->d_set, words)));
    CK(h, cudaMemcpyAsync(h->d_set, set, words * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
  }
  int32_t *d_count = h->d_hr, *d_failed = d_count + cells;
  const int grid = (n + HEADROOM_THREADS - 1) / HEADROOM_THREADS;
  for (int s = 0; s < n_shapes && n > 0; s++) {
    const int C = c_off[s + 1] - c_off[s];
    const egs_unit *u = units + c_off[s];
    by_geometry(h, [&](auto W) -> int {
      constexpr int G = decltype(W)::G, NP = decltype(W)::NP;
      HeadroomArgsT<ReqOf<NP>> a;
      a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total;
      a.node0 = node0; a.n = n; a.policy = h->policy; a.limit = limit;
      a.req = make_req<ReqOf<NP>>(C, u); a.t = table(h, slots[s]);
      a.count = d_count + (size_t)s * n; a.failed = d_failed + (size_t)s * n; a.summary = h->d_hr_sum + (size_t)s * 4;
      const NodeSet ns{set ? h->d_set.get() : nullptr};
      const bool single = is_single(C, u);
      if (set && single) k_headroom<G, NP, true, true><<<grid, HEADROOM_THREADS, 0, h->stream>>>(a, ns);
      else if (set) k_headroom<G, NP, false, true><<<grid, HEADROOM_THREADS, 0, h->stream>>>(a, ns);
      else if (single) k_headroom<G, NP, true, false><<<grid, HEADROOM_THREADS, 0, h->stream>>>(a, ns);
      else k_headroom<G, NP, false, false><<<grid, HEADROOM_THREADS, 0, h->stream>>>(a, ns);
      return EGS_OK;
    });
    CK(h, cudaGetLastError());
  }
  TRY(ensure_stage(h, 2 * cells * sizeof(int32_t) + (size_t)n_shapes * 4 * sizeof(int64_t)));
  int64_t *s_sum = (int64_t *)h->h_stage.get();
  int32_t *s_cells = (int32_t *)(s_sum + (size_t)n_shapes * 4);
  CK(h, cudaMemcpyAsync(s_sum, h->d_hr_sum, (size_t)n_shapes * 4 * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
  if (cells) CK(h, cudaMemcpyAsync(s_cells, d_count, 2 * cells * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  if (out_summary) memcpy(out_summary, s_sum, (size_t)n_shapes * 4 * sizeof(int64_t));
  if (out_count) memcpy(out_count, s_cells, cells * sizeof(int32_t));
  if (out_failed) memcpy(out_failed, s_cells + cells, cells * sizeof(int32_t));
  return EGS_OK;
}

// ------------------------------------------------------------------------------- eviction what-if
// Every argument is checked before the shape is interned or anything is staged.  The podsMap decisions are taken on
// the host, read-only; only the victims that apply reach the device.  One k_evict launch and one synchronisation.
extern "C" int egs_evict_fit(egs_handle *h, int n_containers, const egs_unit *units, int n, const int32_t *node_ids,
                             const int32_t *victim_off, const egs_mutation *victims, int32_t *out_status,
                             int32_t *out_score, uint8_t *out_alloc_mask) {
  if (!h) return EGS_ERR_BAD_ARG;
  Guard g(h);
  if (n < 0 || (n > 0 && (!node_ids || !out_status || !out_score || !out_alloc_mask)))
    return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: n >= 0 candidate nodes, and node_ids and all three outputs");
  const int urc = check_units(n_containers, units, h->c_max);      // what egs_filter returns for it
  if (urc != EGS_OK) return fail(h, urc, "egs_evict_fit: malformed pending pod");
  if (leaf_split(h, n_containers, units))
    return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: shapes Traded by the leaf-split kernels (more than 2^12 leaves) are not served");
  for (int j = 0; j < n; j++) {
    const int rc = check_node(h, node_ids[j]);
    if (rc != EGS_OK) return fail(h, rc, "egs_evict_fit: candidate node out of range or not set");
    if (h->world > 1 && (node_ids[j] < h->lo || node_ids[j] >= h->hi))
      return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: on a sharded handle every node must lie inside the rank's egs_shard_range");
  }
  std::vector<int32_t> sorted(node_ids, node_ids + n);
  std::sort(sorted.begin(), sorted.end());
  if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
    return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: a candidate node repeated");
  if (victim_off) {
    if (victim_off[0] != 0) return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: victim_off[0] != 0");
    for (int j = 0; j < n; j++)
      if (victim_off[j + 1] < victim_off[j]) return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: victim_off decreases");
    if (victim_off[n] > 0 && !victims) return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: victims missing");
    for (int j = 0; j < n; j++)
      for (int k = victim_off[j]; k < victim_off[j + 1]; k++) {
        const egs_mutation &m = victims[k];
        if (m.kind != EGS_MUT_FORGET || m.node_id != node_ids[j])
          return fail(h, EGS_ERR_BAD_ARG, "egs_evict_fit: a victim is an EGS_MUT_FORGET record of its candidate node");
        const int rc = check_record(h, m);
        if (rc != EGS_OK) return fail(h, rc, "egs_evict_fit: a victim record egs_mutations_apply refuses");
      }
  }
  int slot;
  TRY(intern(h, n_containers, units, &slot));
  if (n == 0) return EGS_OK;
  TRY(settle_pending(h, true));                   // the podsMap decisions need every batch's binds in the book
  const size_t sn = (size_t)n, ab = (size_t)h->planes * h->mask_b;   // alloc bytes per node
  if (sn > h->d_ids.cap()) {
    const size_t cap = std::max(sn, (size_t)4096);
    CK(h, grow(h->stream, false, to(h->d_ids, cap), to(h->d_fit, cap), to(h->d_score, cap)));
  }
  TRY(ensure_out(h, n));
  return by_geometry(h, [&](auto W) -> int {
    constexpr int G = decltype(W)::G, NP = decltype(W)::NP;
    typedef ApplyOp<G> Op;
    // the victims that apply: in the node's podsMap and not forgotten by an earlier victim of the same list
    std::vector<Op> ops;
    std::vector<int32_t> off(sn + 1, 0);
    std::vector<uint64_t> gone;
    for (int j = 0; j < n; j++) {
      off[j] = (int32_t)ops.size();
      gone.clear();
      for (int k = victim_off ? victim_off[j] : 0; victim_off && k < victim_off[j + 1]; k++) {
        const egs_mutation &m = victims[k];
        if (!h->book.in_pods_map(m.node_id, m.uid) || std::find(gone.begin(), gone.end(), m.uid) != gone.end()) continue;
        gone.push_back(m.uid);
        ops.push_back(apply_op_of<G>(m, 1));
      }
    }
    off[sn] = (int32_t)ops.size();
    const size_t nd = ops.size();
    if (nd * sizeof(Op) > h->d_ops.cap() || sn + 1 > h->d_group_off.cap()) {
      const size_t cap = std::max({nd, sn, (size_t)1024, h->d_ops.cap() / sizeof(Op)});
      CK(h, grow(h->stream, false, to(h->d_ops, cap * sizeof(Op)), to(h->d_group_off, cap + 1)));
    }
    TRY(ensure_stage(h, std::max(nd * sizeof(Op) + (2 * sn + 1) * sizeof(int32_t), sn * (8 + ab))));
    CK(h, cudaStreamSynchronize(h->stream));     // staging buffer reuse
    Op *so = (Op *)h->h_stage.get();
    int32_t *sid = (int32_t *)(so + nd), *soff = sid + sn;
    std::copy(ops.begin(), ops.end(), so);
    memcpy(sid, node_ids, sn * sizeof(int32_t));
    memcpy(soff, off.data(), (sn + 1) * sizeof(int32_t));
    if (nd) CK(h, cudaMemcpyAsync(h->d_ops, so, nd * sizeof(Op), cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(h->d_ids, sid, sn * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(h->d_group_off, soff, (sn + 1) * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    EvictArgsT<G, ReqOf<NP>> a;
    a.core = h->d_core; a.mem = h->d_mem; a.mem_total = h->d_mem_total;
    a.n = n; a.policy = h->policy; a.req = make_req<ReqOf<NP>>(n_containers, units); a.t = table(h, slot);
    a.ids = h->d_ids; a.off = h->d_group_off; a.ops = (const Op *)h->d_ops.get();
    a.status = h->d_o_status; a.score = h->d_score; a.alloc = h->d_o_alloc;
    const int grid = (n + EVICT_THREADS - 1) / EVICT_THREADS;
    if (is_single(n_containers, units)) k_evict<G, NP, true><<<grid, EVICT_THREADS, 0, h->stream>>>(a);
    else k_evict<G, NP, false><<<grid, EVICT_THREADS, 0, h->stream>>>(a);
    CK(h, cudaGetLastError());
    // back through the staging buffer, after the copies out of it in stream order
    char *s = h->h_stage.get();
    CK(h, cudaMemcpyAsync(s, h->d_o_status, sn * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(s + 4 * sn, h->d_score, sn * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(s + 8 * sn, h->d_o_alloc, sn * ab, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    memcpy(out_status, s, sn * sizeof(int32_t));
    memcpy(out_score, s + 4 * sn, sn * sizeof(int32_t));
    memcpy(out_alloc_mask, s + 8 * sn, sn * ab);
    return EGS_OK;
  });
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
  if (is_sidecar(h)) return fail(h, EGS_ERR_BAD_ARG, "the sharded engine is the rounds engine: it needs c_max <= EGS_MAX_CONTAINERS");
  checkpoint_free(h);                             // a checkpoint holds for the shard layout it was taken under
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
  if (n_containers > EGS_C && n_containers <= h->c_max)
    return fail(h, EGS_ERR_BAD_ARG, "egs_profile_evaluate takes at most EGS_MAX_CONTAINERS containers");
  TRY(check_units(n_containers, units));
  const size_t np = (size_t)h->n_pad;
  if (!h->d_ev_fit) CK(h, grow(h->stream, false, to(h->d_ev_fit, np), to(h->d_ev_score, np), to(h->d_ev_gpu, np * EGS_C * h->mask_b)));
  const size_t flush_bytes = (size_t)256 << 20;
  if (flush_l2 && !h->d_flush) CK(h, grow(h->stream, false, to(h->d_flush, flush_bytes)));
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
    by_geometry(h, [&](auto W) -> int {
      constexpr int G = decltype(W)::G;
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
