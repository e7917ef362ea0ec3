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
//   k_headroom : egs_headroom, per node of a range the binds a stream of pods of one shape would make (read-only).
//   k_evict    : egs_evict_fit, per candidate node whether a pending pod fits once the node's victims are gone
//                (read-only).
//   k_trade_probe / k_trade_leaves / k_trade_commit : the leaf-split Trade of a sidecar handle (c_max > 4) for shapes
//                whose leaf space is larger than one thread should walk; the kernels above then only read caches.
// Every kernel here is a template on the geometry: row width G (8, or 16 on a handle with g_max > 8) and, where masks
// or requests are involved, NP mask planes per pod (4, or 8 on a sidecar handle).  The rounds engine (egs_rounds.cuh)
// uses the (8, 4) instantiations only.
#pragma once
#include "egs_device.cuh"

#define PASS_THREADS 256

struct OptTable {            // option cache of ONE request shape (slot)
  uint8_t *st;               // [N_pad]  OPT_*
  int32_t *sc;               // [N_pad]  option.Score
  uint8_t *al;               // [NP][N_pad] MaskT<G> GPU mask per container (option.Allocated)
  size_t plane;              // N_pad
};

struct Partial { unsigned long long key, fd, sd; int fit; int pad; };

struct PodOut {              // per-pod outputs of the batch loop (device pointers, may be null)
  int32_t *node, *status, *fit_count;
  uint8_t *alloc;            // [P][NP] MaskT<G>
  unsigned long long *fit_digest, *score_digest;
};

// A candidate node set of egs_schedule_batch_nodes on the device: bit n & 63 of word n >> 6 admits node n.  The
// masked kernels (k_pass_nodes, k_evaluate_nodes, k_trade_probe_nodes, k_select_nodes) share their body with the
// unmasked ones through a MASKED template flag; with MASKED false the set is never read.
struct NodeSet {
  const uint64_t *w;
  __device__ __forceinline__ bool admits(int i) const { return (w[i >> 6] >> (i & 63)) & 1ull; }
};

// The six per-pod outputs of pod p; `masks` packs the NP alloc masks of the pod (one MaskT<G> per container).
template <int G, int NP = EGS_C>
__device__ __forceinline__ void write_pod_out(const PodOut &o, int p, int node, int status, int fit, unsigned long long fd,
                                              unsigned long long sd, PackedT<G, NP> masks) {
  static_assert(NP * sizeof(MaskT<G>) == sizeof(PackedT<G, NP>), "alloc row == one packed word");
  if (o.node) o.node[p] = node;
  if (o.status) o.status[p] = status;
  if (o.fit_count) o.fit_count[p] = fit;
  if (o.fit_digest) o.fit_digest[p] = fd;
  if (o.score_digest) o.score_digest[p] = sd;
  if (o.alloc) reinterpret_cast<PackedT<G, NP> *>(o.alloc)[p] = masks;
}

template <class R>
struct PassArgsT {
  const int32_t *core, *mem, *mem_total;   // rows are written by the bind in the last block
  int32_t *core_w, *mem_w;
  int n, policy;
  R req;
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
template <int G, bool SINGLE, class R>
__device__ __forceinline__ uint8_t assume_option(const OptTable &t, size_t i, const int32_t *core, const int32_t *mem,
                                                 const int32_t *mem_total, const R &req, int policy, int &score) {
  uint8_t st = t.st[i];
  if (st == OPT_CACHED) { score = t.sc[i]; return st; }
  if (st != OPT_ABSENT) return st;
  int c[G], m[G]; PackedT<G, R::NC> masks;
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
template <int G, int NP = EGS_C>
__device__ __forceinline__ PackedT<G, NP> option_masks(const OptTable &t, size_t w, int C) {
  PackedT<G, NP> masks = 0;
  for (int c = 0; c < C; c++) masks |= (PackedT<G, NP>)reinterpret_cast<const MaskT<G> *>(t.al)[(size_t)c * t.plane + w] << (G * c);
  return masks;
}

// NodeAllocator.Allocate (node.go:87-104) of node w's cached option; one thread.  The entry goes before the Transact
// (deferred delete, node.go:90-92); the rows changed, so the node's UNFIT memos go too.
template <int G, class R>
__device__ __forceinline__ int allocate_option(const OptTable &t, size_t w, int32_t *core, int32_t *mem, int mem_total,
                                               const R &req, uint8_t *all_st, size_t slot_stride, int n_slots,
                                               PackedT<G, R::NC> &masks) {
  masks = option_masks<G, R::NC>(t, w, req.C);
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
// k_pass_nodes: the same for a pod restricted to a node set -- an excluded node takes no Assume and counts nowhere.
template <int G, int NP, bool SINGLE, bool MASKED>
__device__ __forceinline__ void pass_body(const PassArgsT<ReqOf<NP>> &a, NodeSet set) {
  __shared__ Partial sm[PASS_THREADS / 32];
  __shared__ bool is_last;
  const int i = blockIdx.x * PASS_THREADS + threadIdx.x;
  unsigned long long key = 0, fd = 0, sd = 0;
  int fit = 0;
  if (i < a.n && (!MASKED || set.admits(i))) {
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
    PackedT<G, NP> masks = 0;
    if (key != 0) {
      node = (int)key_node(key);
      status = allocate_option<G>(a.t, (size_t)node, a.core_w, a.mem_w, a.mem_total[node], a.req, a.all_st, a.slot_stride,
                               a.n_slots, masks);
      if (status != EGS_OK) masks = 0;
    }
    write_pod_out<G, NP>(a.out, a.pod, node, status, fit, fd, sd, masks);
  }
}
template <int G, int NP, bool SINGLE>
__global__ void __launch_bounds__(PASS_THREADS, G > EGS_G ? 1 : 0) k_pass(PassArgsT<ReqOf<NP>> a) {
  pass_body<G, NP, SINGLE, false>(a, NodeSet{nullptr});
}
template <int G, int NP, bool SINGLE>
__global__ void __launch_bounds__(PASS_THREADS, G > EGS_G ? 1 : 0) k_pass_nodes(PassArgsT<ReqOf<NP>> a, NodeSet set) {
  pass_body<G, NP, SINGLE, true>(a, set);
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

// k_evaluate_nodes (the cold fill of a batch under a node set): an excluded node is neither read nor written.
template <int G, bool SINGLE, int ITEMS, bool MASKED>
__device__ __forceinline__ void evaluate_body(const EvalArgs &a, NodeSet set) {
  const int base = blockIdx.x * (256 * ITEMS) + threadIdx.x;
  int c[ITEMS][G], m[ITEMS][G];
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    const int j = base + it * 256;
    if (j < a.n && (!MASKED || set.admits(a.lo + j))) load_row(a.core, a.mem, (size_t)(a.lo + j), c[it], m[it]);
  }
#pragma unroll
  for (int it = 0; it < ITEMS; it++) {
    const int j = base + it * 256;
    if (j >= a.n || (MASKED && !set.admits(a.lo + j))) continue;
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
template <int G, bool SINGLE, int ITEMS>
__global__ void __launch_bounds__(256) k_evaluate(EvalArgs a) { evaluate_body<G, SINGLE, ITEMS, false>(a, NodeSet{nullptr}); }
template <int G, bool SINGLE, int ITEMS>
__global__ void __launch_bounds__(256) k_evaluate_nodes(EvalArgs a, NodeSet set) { evaluate_body<G, SINGLE, ITEMS, true>(a, set); }

// --------------------------------------------------------------------------------------------
// verbs over an explicit candidate list (ids == nullptr -> identity)
// --------------------------------------------------------------------------------------------
template <class R>
struct GatherArgsT {
  const int32_t *core, *mem, *mem_total;
  int n, n_nodes, policy;
  R req;
  OptTable t;
  const int32_t *ids;
  uint8_t *out_fit; int32_t *out_score; int *panic_flag;
};

// Assume per node (node.go:61-73)
template <int G, int NP, bool SINGLE>
__global__ void __launch_bounds__(256) k_gather_filter(GatherArgsT<ReqOf<NP>> a) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n) return;
  const int i = a.ids ? a.ids[j] : j;
  if (i < 0 || i >= a.n_nodes) { a.out_fit[j] = 0; return; }
  int score;
  a.out_fit[j] = assume_option<G, SINGLE>(a.t, (size_t)i, a.core, a.mem, a.mem_total, a.req, a.policy, score) == OPT_CACHED;
}

// Score per node (node.go:75-85): cached score; no entry -> Assume; fails -> 0, succeeds -> the
// reference dereferences nil (panic) -- flagged.
template <int G, int NP, bool SINGLE>
__global__ void __launch_bounds__(256) k_gather_score(GatherArgsT<ReqOf<NP>> a) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= a.n) return;
  const int i = a.ids ? a.ids[j] : j;
  if (i < 0 || i >= a.n_nodes) { a.out_score[j] = 0; return; }   // scheduler.go:176-179
  if (a.t.st[i] == OPT_CACHED) { a.out_score[j] = a.t.sc[i]; return; }
  int score;                                                       // Assume caches the option before the nil deref
  if (assume_option<G, SINGLE>(a.t, (size_t)i, a.core, a.mem, a.mem_total, a.req, a.policy, score) == OPT_CACHED) *a.panic_flag = 1;
  a.out_score[j] = 0;
}

template <class R>
struct BindArgsT {
  int32_t *core, *mem; const int32_t *mem_total;
  int node; R req; OptTable t;
  uint8_t *all_st; size_t slot_stride; int n_slots;
  int skip_transact;          // uid already in the node's podsMap (node.go:149)
  int consume;                // 1: Bind (delete the entry); 0: peek
  int32_t *result;            // [0] had entry, [1] status, [2] masks (low 32 bits), [3] score, [4] masks >> 32 (64-bit word)
};
template <int G, int NP>
__global__ void k_bind(BindArgsT<ReqOf<NP>> a) {
  const size_t w = (size_t)a.node;
  const bool had = a.t.st[w] == OPT_CACHED;
  PackedT<G, NP> masks = 0; int status = EGS_ERR_NO_OPTION, score = 0;
  if (had) {
    score = a.t.sc[w];
    status = EGS_OK;
    if (a.consume && !a.skip_transact) {
      status = allocate_option<G>(a.t, w, a.core, a.mem, a.mem_total[w], a.req, a.all_st, a.slot_stride, a.n_slots, masks);
    } else {                                     // peek, or Bind of a known uid (node.go:149): the entry goes, rows stay
      masks = option_masks<G, NP>(a.t, w, a.req.C);
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

// --------------------------------------------------------------------------------------------
// k_headroom (egs_headroom): nodes [node0, node0 + n) against one shape, one thread per node running headroom_node on
// a copy of its row and its option entry; nothing is written but the outputs.  Per node count[j] / failed[j]; the four
// sums of summary (binds, nodes with a bind, failed binds, nodes stopped by the limit) are folded per block and added
// with one 64-bit atomicAdd per block and value: integer sums, so the result does not depend on the block order.
// MASKED: a node outside the set is not read and counts 0; with MASKED false the set is never read.
// --------------------------------------------------------------------------------------------
#define HEADROOM_THREADS 256
template <class R>
struct HeadroomArgsT {
  const int32_t *core, *mem, *mem_total;
  int node0, n, policy, limit;
  R req;
  OptTable t;
  int32_t *count, *failed;                  // [n] each, may be null
  unsigned long long *summary;              // [4]
};
// At G = 16 a minimum of one block per SM lifts ptxas's default register cap, as for k_pass.
template <int G, int NP, bool SINGLE, bool MASKED>
__global__ void __launch_bounds__(HEADROOM_THREADS, G > EGS_G ? 1 : 0) k_headroom(HeadroomArgsT<ReqOf<NP>> a, NodeSet set) {
  __shared__ unsigned long long sm[4][HEADROOM_THREADS / 32];
  const int j = blockIdx.x * HEADROOM_THREADS + threadIdx.x;
  Headroom r = {0, 0, 0};
  if (j < a.n) {
    const int i = a.node0 + j;
    const uint8_t st = (!MASKED || set.admits(i)) ? a.t.st[i] : (uint8_t)OPT_UNFIT;
    if (st != OPT_UNFIT) {
      int c[G], m[G];
      load_row(a.core, a.mem, (size_t)i, c, m);
      const PackedT<G, NP> masks = st == OPT_CACHED ? option_masks<G, NP>(a.t, (size_t)i, a.req.C) : 0;
      r = headroom_node(c, m, SINGLE ? 0 : a.mem_total[i], a.req, SINGLE, a.policy, st, masks, a.limit);
    }
    if (a.count) a.count[j] = r.ok;
    if (a.failed) a.failed[j] = r.failed;
  }
  unsigned long long v[4] = {(unsigned long long)r.ok, r.ok > 0 ? 1ull : 0ull, (unsigned long long)r.failed,
                             (unsigned long long)r.capped};
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    v[k] = warp_sum_u64(v[k]);
    if (lane == 0) sm[k][w] = v[k];
  }
  __syncthreads();
  if (threadIdx.x < 4) {
    unsigned long long s = 0;
    for (int q = 0; q < HEADROOM_THREADS / 32; q++) s += sm[threadIdx.x][q];
    if (s) atomicAdd(a.summary + threadIdx.x, s);
  }
}

// --------------------------------------------------------------------------------------------
// k_evict (egs_evict_fit): one thread per candidate node ids[j], running evict_node on a copy of its row and its option
// entry with the victims that apply there, ops[off[j] .. off[j+1]) (the host took the podsMap decisions).  Nothing is
// written but the outputs: status[j], score[j] and the packed masks alloc[j].
// --------------------------------------------------------------------------------------------
#define EVICT_THREADS 256
template <int G, class R>
struct EvictArgsT {
  const int32_t *core, *mem, *mem_total;
  int n, policy;
  R req;
  OptTable t;
  const int32_t *ids, *off;                 // [n] candidate nodes, [n + 1] offsets into ops
  const ApplyOp<G> *ops;                    // cancel == 1 each
  int32_t *status, *score;                  // [n]
  uint8_t *alloc;                           // [n] packed words of NP MaskT<G>
};
// At G = 16 a minimum of one block per SM lifts ptxas's default register cap, as for k_pass.
template <int G, int NP, bool SINGLE>
__global__ void __launch_bounds__(EVICT_THREADS, G > EGS_G ? 1 : 0) k_evict(EvictArgsT<G, ReqOf<NP>> a) {
  const int j = blockIdx.x * EVICT_THREADS + threadIdx.x;
  if (j >= a.n) return;
  const size_t i = (size_t)a.ids[j];
  const uint8_t st = a.t.st[i];
  int c[G], m[G];
  load_row(a.core, a.mem, i, c, m);
  int score = st == OPT_CACHED ? a.t.sc[i] : 0;
  PackedT<G, NP> masks = st == OPT_CACHED ? option_masks<G, NP>(a.t, i, a.req.C) : 0;
  const int o0 = a.off[j];
  const int status = evict_node(c, m, a.mem_total[i], a.req, SINGLE, a.policy, st, a.ops + o0, a.off[j + 1] - o0, score,
                                masks);
  a.status[j] = status;
  a.score[j] = score;
  reinterpret_cast<PackedT<G, NP> *>(a.alloc)[j] = masks;
}

// --------------------------------------------------------------------------------------------
// Leaf-split Trade (sidecar handles, geometry (8, 8)): the Trade of every node whose option is absent, with the leaf
// space of each node (trade_leaf_eval: one digit per branching container, `bits` wide) cut into chunks of LEAF_CHUNK
// leaves spread over the whole GPU.  Three launches on the handle's stream, no host synchronisation:
//   k_trade_probe  : candidates whose state is OPT_ABSENT go to a miss list (count on the device); with out_score it
//                    is also Score's read of the cache (cached score, else 0).
//   k_trade_leaves : grid-strides over (miss, tile of LEAF_THREADS chunks); each thread walks its chunk in leaf order,
//                    skipping every leaf whose prefix is already infeasible; one 64-bit atomicMax per CTA and miss on
//                    key = score << 32 | (leaf + 1), so key 0 is "no feasible leaf" and the max over keys is "the last
//                    maximal leaf wins" (gpu.go:85).  Scores stay below 2^31: each of up to 8 sentinel units adds 1
//                    to a GPU, so range <= (2^25 + 8 + 2^20 + 8) / 2 < 2^24.1 and range * 100 < 2^30.8.
//   k_trade_commit : decodes each miss's winning leaf into its masks and caches the option, or memoises OPT_UNFIT.
// --------------------------------------------------------------------------------------------
#define LEAF_THREADS 256
#define LEAF_CHUNK 64

struct LeafArgs {
  const int32_t *core, *mem, *mem_total;
  int policy, bits, nbranch, tiles;         // tiles: ceil(nleaf / (LEAF_THREADS * LEAF_CHUNK)) per miss
  ReqW req;
  int32_t *miss; unsigned int *n_miss; unsigned long long *keys;
};

struct ProbeArgs {
  const uint8_t *st; const int32_t *sc;
  const int32_t *ids; int n, n_nodes;       // ids == nullptr -> identity
  int32_t *miss; unsigned int *n_miss; unsigned long long *keys;
  int32_t *out_score;                       // optional: Score's reads (node.go:75-85)
};

// k_trade_probe_nodes (a batch under a node set): an excluded node is no miss.
template <bool MASKED>
__device__ __forceinline__ void probe_body(ProbeArgs a, NodeSet set) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int i = j < a.n ? (a.ids ? a.ids[j] : j) : -1;
  const bool valid = i >= 0 && i < a.n_nodes;
  const uint8_t st = valid ? a.st[i] : (uint8_t)OPT_UNFIT;
  if (a.out_score && j < a.n) a.out_score[j] = st == OPT_CACHED ? a.sc[i] : 0;
  const bool miss = st == OPT_ABSENT && (!MASKED || set.admits(i));
  const unsigned b = __ballot_sync(0xffffffffu, miss);       // one atomic per warp
  if (!b) return;
  const int lane = threadIdx.x & 31, lead = __ffs(b) - 1;
  unsigned base = 0;
  if (lane == lead) base = atomicAdd(a.n_miss, (unsigned)__popc(b));
  base = __shfl_sync(0xffffffffu, base, lead);
  if (miss) {
    const unsigned m = base + __popc(b & ((1u << lane) - 1u));
    a.miss[m] = i; a.keys[m] = 0ull;
  }
}
__global__ void __launch_bounds__(256) k_trade_probe(ProbeArgs a) { probe_body<false>(a, NodeSet{nullptr}); }
__global__ void __launch_bounds__(256) k_trade_probe_nodes(ProbeArgs a, NodeSet set) { probe_body<true>(a, set); }

__global__ void __launch_bounds__(LEAF_THREADS) k_trade_leaves(LeafArgs a) {
  __shared__ unsigned long long sm[LEAF_THREADS / 32];
  const unsigned long long items = (unsigned long long)*a.n_miss * (unsigned)a.tiles;
  const int nleaf = 1 << (a.bits * a.nbranch);
  for (unsigned long long t = blockIdx.x; t < items; t += gridDim.x) {
    const int m = (int)(t / (unsigned)a.tiles), tile = (int)(t % (unsigned)a.tiles);
    const size_t node = (size_t)a.miss[m];
    int c[EGS_G], mm[EGS_G];
    load_row(a.core, a.mem, node, c, mm);
    const int mt = a.mem_total[node];
    int leaf = (tile * LEAF_THREADS + (int)threadIdx.x) * LEAF_CHUNK;
    const int end = EGS_MIN(leaf + LEAF_CHUNK, nleaf);
    unsigned long long best = 0;
    while (leaf < end) {
      uint64_t mk; int fail;
      const int s = trade_leaf_eval(c, mm, mt, a.req, a.policy, a.bits, a.nbranch, leaf, mk, &fail);
      if (s >= 0) {
        const unsigned long long key = ((unsigned long long)(uint32_t)s << 32) | (unsigned)(leaf + 1);
        best = key > best ? key : best;
        leaf++;
      } else {
        leaf = trade_leaf_next(leaf, fail, a.bits, a.nbranch);
      }
    }
    best = warp_max_u64(best);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
      best = threadIdx.x < LEAF_THREADS / 32 ? sm[threadIdx.x] : 0ull;
      best = warp_max_u64(best);
      if (threadIdx.x == 0 && best) atomicMax(a.keys + m, best);
    }
    __syncthreads();
  }
}

// One thread per miss.  panic_flag (Score): a node that had no entry and fits is the reference's nil-option panic.
__global__ void __launch_bounds__(256) k_trade_commit(LeafArgs a, OptTable t, int *panic_flag) {
  const int m = blockIdx.x * 256 + threadIdx.x;
  if (m >= (int)*a.n_miss) return;
  const size_t node = (size_t)a.miss[m];
  const unsigned long long key = a.keys[m];
  if (!key) { t.st[node] = OPT_UNFIT; return; }
  int c[EGS_G], mm[EGS_G];
  load_row(a.core, a.mem, node, c, mm);
  uint64_t masks = 0;
  const int leaf = (int)(uint32_t)key - 1;
  trade_leaf_eval(c, mm, a.mem_total[node], a.req, a.policy, a.bits, a.nbranch, leaf, masks);
  t.sc[node] = (int32_t)(key >> 32);
  for (int k = 0; k < a.req.C; k++) t.al[(size_t)k * t.plane + node] = (uint8_t)(masks >> (EGS_G * k));
  t.st[node] = OPT_CACHED;
  if (panic_flag) *panic_flag = 1;
}
