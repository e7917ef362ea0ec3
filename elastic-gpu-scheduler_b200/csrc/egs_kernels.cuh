// egs_kernels.cuh -- sm_90a kernels of the scheduler core (integer / indexing work only;
// HBM- and latency-bound, no tensor cores).
//
//   k_evaluate : the FULL-EVALUATE ("score") kernel -- Trade on every node, no cache shortcut.
//                Roofline kernel: reads 2*G*4 B of rows, writes fit(1)+score(4)+gpu(C) per node.
//   k_pass     : one pod against all nodes honouring the option cache (node.go:61-85), with
//                fit/score digests, first-max selection and the bind (node.go:87-104) fused in
//                the last block.  EGS_MODE_RESCAN launches it once per pod.
//   k_gather_* : /scheduler/filter and /scheduler/priorities over an explicit candidate list.
//   k_bind / k_apply : single-node mutations (Bind, AddPod, ForgetPod); k_apply_many: many AddPod /
//                ForgetPod in one launch.
// Each reference step these kernels share is written once: Assume (assume_option), Allocate
// (allocate_option), and the AddPod / ForgetPod row update (apply_op, egs_device.cuh).
// Every kernel here is a template on the row width G (8, or 16 on a handle with g_max > 8); the rounds engine
// (egs_rounds.cuh) uses the 8-wide instantiations only.
#pragma once
#include "egs_device.cuh"

#define PASS_THREADS 256

struct OptTable {            // option cache of ONE request shape (slot)
  uint8_t *st;               // [N_pad]  OPT_*
  int32_t *sc;               // [N_pad]  option.Score
  uint8_t *al;               // [EGS_C][N_pad] MaskT<G> GPU mask per container (option.Allocated)
  size_t plane;              // N_pad
};

struct Partial { unsigned long long key, fd, sd; int fit; int pad; };

struct PodOut {              // per-pod outputs of the batch loop (device pointers, may be null)
  int32_t *node, *status, *fit_count;
  uint8_t *alloc;            // [P][EGS_C] MaskT<G>
  unsigned long long *fit_digest, *score_digest;
};

// The six per-pod outputs of pod p; `masks` packs the EGS_C alloc masks of the pod (one MaskT<G> per container).
template <int G>
__device__ __forceinline__ void write_pod_out(const PodOut &o, int p, int node, int status, int fit, unsigned long long fd,
                                              unsigned long long sd, PackedT<G> masks) {
  static_assert(EGS_C * sizeof(MaskT<G>) == sizeof(PackedT<G>), "alloc row == one packed word");
  if (o.node) o.node[p] = node;
  if (o.status) o.status[p] = status;
  if (o.fit_count) o.fit_count[p] = fit;
  if (o.fit_digest) o.fit_digest[p] = fd;
  if (o.score_digest) o.score_digest[p] = sd;
  if (o.alloc) reinterpret_cast<PackedT<G> *>(o.alloc)[p] = masks;
}

struct PassArgs {
  const int32_t *core, *mem, *mem_total;   // rows are written by the bind in the last block
  int32_t *core_w, *mem_w;
  int n, policy;
  Req req;
  OptTable t;
  uint8_t *all_st; size_t slot_stride; int n_slots;   // every slot's state plane (UNFIT memo reset)
  uint8_t *vec_fit; int32_t *vec_score;    // optional full vectors
  Partial *partials; unsigned int *ticket;
  int pod; PodOut out;
};

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { unsigned long long x = __shfl_xor_sync(0xffffffffu, v, o); v = x > v ? x : v; }
  return v;
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i32(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide reduction of (max key, sum fd, sum sd, sum fit); result valid in thread 0
__device__ __forceinline__ void block_reduce(unsigned long long &key, unsigned long long &fd,
                                             unsigned long long &sd, int &fit, Partial *sm) {
  key = warp_max_u64(key); fd = warp_sum_u64(fd); sd = warp_sum_u64(sd); fit = warp_sum_i32(fit);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  if (lane == 0) { sm[w].key = key; sm[w].fd = fd; sm[w].sd = sd; sm[w].fit = fit; }
  __syncthreads();
  if (w == 0) {
    key = lane < nw ? sm[lane].key : 0ull; fd = lane < nw ? sm[lane].fd : 0ull;
    sd = lane < nw ? sm[lane].sd : 0ull; fit = lane < nw ? sm[lane].fit : 0;
    key = warp_max_u64(key); fd = warp_sum_u64(fd); sd = warp_sum_u64(sd); fit = warp_sum_i32(fit);
  }
  __syncthreads();
}

// Rows of node w changed: every UNFIT memo of that node is stale (the reference would re-Trade).
__device__ __forceinline__ void memo_reset(uint8_t *all_st, size_t slot_stride, int n_slots, size_t w) {
  for (int s = 0; s < n_slots; s++) {
    uint8_t *p = all_st + (size_t)s * slot_stride + w;
    if (*p == OPT_UNFIT) *p = OPT_ABSENT;
  }
}

// NodeAllocator.Assume (node.go:61-73) on node i; one thread.  An entry is reused without re-validation
// (node.go:64-66); no entry -> Trade (node.go:67-71): the option is cached, or the failure memoised as UNFIT (the
// reference caches nothing then and re-Trades with the same outcome).  Returns the state after Assume; `score` is
// set when it is OPT_CACHED.  The fast Trade ignores mem_total, so SINGLE does not load it.
template <int G, bool SINGLE>
__device__ __forceinline__ uint8_t assume_option(const OptTable &t, size_t i, const int32_t *core, const int32_t *mem,
                                                 const int32_t *mem_total, const Req &req, int policy, int &score) {
  uint8_t st = t.st[i];
  if (st == OPT_CACHED) { score = t.sc[i]; return st; }
  if (st != OPT_ABSENT) return st;
  int c[G], m[G]; PackedT<G> masks;
  load_row(core, mem, i, c, m);
  if (trade_any(c, m, SINGLE ? 0 : mem_total[i], req, SINGLE, policy, score, masks)) {
    st = OPT_CACHED;
    t.sc[i] = score;
    for (int k = 0; k < req.C; k++) reinterpret_cast<MaskT<G> *>(t.al)[(size_t)k * t.plane + i] = (MaskT<G>)(masks >> (G * k));
  } else {
    st = OPT_UNFIT;
  }
  t.st[i] = st;
  return st;
}

// GPU masks of node w's option, one MaskT<G> per container.
template <int G>
__device__ __forceinline__ PackedT<G> option_masks(const OptTable &t, size_t w, int C) {
  PackedT<G> masks = 0;
  for (int c = 0; c < C; c++) masks |= (PackedT<G>)reinterpret_cast<const MaskT<G> *>(t.al)[(size_t)c * t.plane + w] << (G * c);
  return masks;
}

// NodeAllocator.Allocate (node.go:87-104) of node w's cached option; one thread.  The entry goes before the Transact
// (deferred delete, node.go:90-92); the rows changed, so the node's UNFIT memos go too.
template <int G>
__device__ __forceinline__ int allocate_option(const OptTable &t, size_t w, int32_t *core, int32_t *mem, int mem_total,
                                               const Req &req, uint8_t *all_st, size_t slot_stride, int n_slots,
                                               PackedT<G> &masks) {
  masks = option_masks<G>(t, w, req.C);
  t.st[w] = OPT_ABSENT;
  const bool ok = transact_row<G>(core + w * G, mem + w * G, mem_total, req, masks);
  memo_reset(all_st, slot_stride, n_slots, w);
  return ok ? EGS_OK : EGS_ERR_TRANSACT;
}

// --------------------------------------------------------------------------------------------
// k_pass: one pod, all nodes.  One thread per node; block partials; the last block to finish
// (atomic ticket) folds the partials, picks the first max and binds it.
// --------------------------------------------------------------------------------------------
// At G = 16 a minimum of one block per SM lifts ptxas's default 64-register cap, under which the 16-wide row spills
// (70 / 80 registers without spills, sm_90a); 0 leaves the 8-wide instantiations exactly as they were.
template <int G, bool SINGLE>
__global__ void __launch_bounds__(PASS_THREADS, G > EGS_G ? 1 : 0) k_pass(PassArgs a) {
  __shared__ Partial sm[PASS_THREADS / 32];
  __shared__ bool is_last;
  const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
  unsigned long long key = 0, fd = 0, sd = 0;
  int fit = 0;
  if (i < a.n) {
    int score = 0;
    if (assume_option<G, SINGLE>(a.t, (size_t)i, a.core, a.mem, a.mem_total, a.req, a.policy, score) == OPT_CACHED) {
      fit = 1; key = cand_key(score, (uint32_t)i); fd = fit_term((uint32_t)i); sd = score_term((uint32_t)i, score);
    }
    if (a.vec_fit) a.vec_fit[i] = (uint8_t)fit;
    if (a.vec_score) a.vec_score[i] = fit ? score : 0;
  }
  block_reduce(key, fd, sd, fit, sm);
  if (threadIdx.x == 0) {
    Partial p; p.key = key; p.fd = fd; p.sd = sd; p.fit = fit; p.pad = 0;
    a.partials[blockIdx.x] = p;
    __threadfence();
    is_last = atomicAdd(a.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  key = 0; fd = 0; sd = 0; fit = 0;
  for (int b = threadIdx.x; b < (int)gridDim.x; b += PASS_THREADS) {
    const volatile Partial *q = a.partials + b;
    unsigned long long k2 = q->key;
    key = k2 > key ? k2 : key; fd += q->fd; sd += q->sd; fit += q->fit;
  }
  block_reduce(key, fd, sd, fit, sm);
  if (threadIdx.x == 0) {
    *a.ticket = 0;
    int node = -1, status = EGS_ERR_NOFIT;
    PackedT<G> masks = 0;
    if (key != 0) {
      node = (int)key_node(key);
      status = allocate_option<G>(a.t, (size_t)node, a.core_w, a.mem_w, a.mem_total[node], a.req, a.all_st, a.slot_stride,
                               a.n_slots, masks);
      if (status != EGS_OK) masks = 0;
    }
    write_pod_out<G>(a.out, a.pod, node, status, fit, fd, sd, masks);
  }
}

// --------------------------------------------------------------------------------------------
// k_evaluate: full evaluate of nodes [0,n) for one request, results to flat output planes.
// ITEMS nodes per thread, strided by the block so every warp-level load instruction covers a
// contiguous 32 x 32 B span; all row loads are issued before any Trade runs.
// --------------------------------------------------------------------------------------------
struct EvalArgs {
  const int32_t *core, *mem, *mem_total;
  int lo, n, policy;                                            // nodes [lo, lo + n)
  Req req;
  uint8_t *fit; int32_t *score; uint8_t *gpu; size_t plane;     // gpu: [C][plane] MaskT<G>; all indexed by node id
  uint8_t v_fit, v_unfit;                                       // byte written for fit / unfit (1/0, or OPT_NEW/OPT_UNFIT
};                                                              // when the target is an option table)

template <int G, bool SINGLE, int ITEMS>
__global__ void __launch_bounds__(256) k_evaluate(EvalArgs a) {
  const int base = blockIdx.x * (256 * ITEMS) + threadIdx.x;
  int c[ITEMS][G], m[ITEMS][G];
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    const int j = base + it * 256;
    if (j < a.n) load_row(a.core, a.mem, (size_t)(a.lo + j), c[it], m[it]);
  }
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    const int j = base + it * 256;
    if (j >= a.n) continue;
    const int i = a.lo + j;
    int score; PackedT<G> masks;
    const int mt = SINGLE ? 0 : a.mem_total[i];
    const bool ok = trade_any(c[it], m[it], mt, a.req, SINGLE, a.policy, score, masks);
    a.fit[i] = ok ? a.v_fit : a.v_unfit;
    a.score[i] = ok ? score : 0;
    MaskT<G> *gpu = reinterpret_cast<MaskT<G> *>(a.gpu);
    if (SINGLE) gpu[i] = ok ? (MaskT<G>)masks : 0;
    else for (int k = 0; k < a.req.C; k++) gpu[(size_t)k * a.plane + i] = ok ? (MaskT<G>)(masks >> (G * k)) : 0;
  }
}

// --------------------------------------------------------------------------------------------
// verbs over an explicit candidate list (ids == nullptr -> identity)
// --------------------------------------------------------------------------------------------
struct GatherArgs {
  const int32_t *core, *mem, *mem_total;
  int n, n_nodes, policy;
  Req req;
  OptTable t;
  const int32_t *ids;
  uint8_t *out_fit; int32_t *out_score; int *panic_flag;
};

// Assume per node (node.go:61-73)
template <int G, bool SINGLE>
__global__ void __launch_bounds__(256) k_gather_filter(GatherArgs a) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n) return;
  const int i = a.ids ? a.ids[j] : j;
  if (i < 0 || i >= a.n_nodes) { a.out_fit[j] = 0; return; }
  int score;
  a.out_fit[j] = assume_option<G, SINGLE>(a.t, (size_t)i, a.core, a.mem, a.mem_total, a.req, a.policy, score) == OPT_CACHED;
}

// Score per node (node.go:75-85): cached score; no entry -> Assume; fails -> 0, succeeds -> the
// reference dereferences nil (panic) -- flagged.
template <int G, bool SINGLE>
__global__ void __launch_bounds__(256) k_gather_score(GatherArgs a) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n) return;
  const int i = a.ids ? a.ids[j] : j;
  if (i < 0 || i >= a.n_nodes) { a.out_score[j] = 0; return; }   // scheduler.go:176-179
  if (a.t.st[i] == OPT_CACHED) { a.out_score[j] = a.t.sc[i]; return; }
  int score;                                                       // Assume caches the option before the nil deref
  if (assume_option<G, SINGLE>(a.t, (size_t)i, a.core, a.mem, a.mem_total, a.req, a.policy, score) == OPT_CACHED) *a.panic_flag = 1;
  a.out_score[j] = 0;
}

struct BindArgs {
  int32_t *core, *mem; const int32_t *mem_total;
  int node; Req req; OptTable t;
  uint8_t *all_st; size_t slot_stride; int n_slots;
  int skip_transact;          // uid already in the node's podsMap (node.go:149)
  int consume;                // 1: Bind (delete the entry); 0: peek
  int32_t *result;            // [0] had entry, [1] status, [2] masks (low 32 bits), [3] score, [4] masks >> 32 (G = 16)
};
template <int G>
__global__ void k_bind(BindArgs a) {
  const size_t w = (size_t)a.node;
  const bool had = a.t.st[w] == OPT_CACHED;
  PackedT<G> masks = 0; int status = EGS_ERR_NO_OPTION, score = 0;
  if (had) {
    score = a.t.sc[w];
    status = EGS_OK;
    if (a.consume && !a.skip_transact) {
      status = allocate_option<G>(a.t, w, a.core, a.mem, a.mem_total[w], a.req, a.all_st, a.slot_stride, a.n_slots, masks);
    } else {                                     // peek, or Bind of a known uid (node.go:149): the entry goes, rows stay
      masks = option_masks<G>(a.t, w, a.req.C);
      if (a.consume) a.t.st[w] = OPT_ABSENT;
    }
  }
  a.result[0] = had; a.result[1] = status; a.result[2] = (int32_t)masks; a.result[3] = score;
  if constexpr (sizeof(masks) > 4) a.result[4] = (int32_t)(masks >> 32);
}

// AddPod / ForgetPod of one pod (apply_op) on node op.node.
template <int G>
struct ApplyArgs {
  int32_t *core, *mem; const int32_t *mem_total;
  ApplyOp<G> op;
  uint8_t *all_st; size_t slot_stride; int n_slots;
};
template <int G>
__global__ void k_apply(ApplyArgs<G> a) {
  const size_t w = (size_t)a.op.node;
  apply_op(a.core + w * G, a.mem + w * G, a.mem_total[w], a.op);
  memo_reset(a.all_st, a.slot_stride, a.n_slots, w);
}

// Many AddPod / ForgetPod row updates in ONE launch: the host has grouped the records by node (record order kept
// inside a node); one thread per touched node applies its run.
template <int G>
struct ApplyManyArgs {
  int32_t *core, *mem; const int32_t *mem_total;
  const ApplyOp<G> *ops; const int32_t *group_off; int n_groups;   // group g = ops[group_off[g] .. group_off[g+1])
  uint8_t *all_st; size_t slot_stride; int n_slots;
};
template <int G>
__global__ void k_apply_many(ApplyManyArgs<G> a) {
  const int gi = blockIdx.x * blockDim.x + threadIdx.x;
  if (gi >= a.n_groups) return;
  const size_t w = (size_t)a.ops[a.group_off[gi]].node;
  for (int o = a.group_off[gi]; o < a.group_off[gi + 1]; o++)
    apply_op(a.core + w * G, a.mem + w * G, a.mem_total[w], a.ops[o]);
  memo_reset(a.all_st, a.slot_stride, a.n_slots, w);
}

// Rows of nodes [node0, node0+n) were overwritten from the host.  full != 0 (node_set: a fresh
// NodeAllocator, node.go:42-50) drops every option; full == 0 (state_load) only clears the UNFIT
// memos -- cached options stay, stale, exactly like the reference's map would.
__global__ void k_node_reset(uint8_t *all_st, size_t slot_stride, int n_slots, int node0, int n, int full) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int s = 0; s < n_slots; s++) {
    uint8_t *p = all_st + (size_t)s * slot_stride + node0 + i;
    if (full || *p == OPT_UNFIT) *p = OPT_ABSENT;
  }
}
