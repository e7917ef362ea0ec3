// egs_rounds.cuh -- EGS_MODE_ROUNDS: the exact round-based decision loop.
//
// Reference semantics (node.go:61-104): a bind changes ONE node's rows and deletes ONE cache
// entry; every other (node, shape) option -- even a stale one -- is by definition unchanged.
// So within a stretch of pods only nodes that WON in that stretch can change.  A round is:
//
//   k_select  (grid, N-proportional, shardable over GPUs): per node and per shape of the
//             round: Trade every absent option (the full-evaluate work), fold fit count and
//             digests, keep the top-32 candidates (score desc, node asc) per CTA and shape.
//   k_merge   (one CTA per shape): fold the per-CTA lists into ONE exact list of up to 128
//             candidates (exact down to the largest 32nd key of a full CTA list), gather each
//             candidate's payload (rows + its options for all round shapes) into the shard's
//             candidate buffer.
//   [ncclAllGather of the candidate buffers when the node list is sharded]
//   k_resolve_mw (ONE CTA, one OWNER WARP per request shape, shared-memory resident): replays the
//             pods in order.  The pods of one shape form a chain that only touches other shapes
//             through the rows of the nodes it binds, so every owner warp prepares its next pod
//             on its own (best tracked option of its shape, its candidate lists, payload prefetch,
//             a speculative Trade of the pending option under the rows' seqlock) and the warps then
//             pass a TICKET in pod order (mbarrier): inside the ticket the speculative Trade is
//             validated (it usually holds) or redone on the current rows, the winner = max(tracked options,
//             best untracked list head) is bound (Transact on the shared-memory copy of the node) and
//             the ticket moves on; outputs, digests and the owner's private tables are updated after
//             the ticket was released.  Stops early when a list runs dry or the tracked table is
//             full; writes the tracked nodes back.
//
// Option states: OPT_NEW marks an option select evaluated AHEAD of the shape's next filter.
// It is only valid while the node's rows stay unchanged; once a pod of that shape has run
// ("observed"), it is an ordinary cached option (OPT_CACHED).
#pragma once
#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <vector>
#include "buffers.h"
#include "egs_kernels.cuh"

#define OPT_NEW 3

#define RK 32        // candidates kept per (CTA, shape) in k_select (one per lane)
#define RQMAX 4      // merged list: up to RQMAX*32 candidates per (shard, shape)
#define RD 8         // shards
#define RSMAX 96     // shapes per round set
#define SEL_THREADS 128
#define SEL_WARPS (SEL_THREADS / 32)
#define MW_MAX_WARPS 16
#define RPROF 32     // resolver cycle counters (-DEGS_RESOLVE_PROF; tools/prof_sections.py names them)

struct RoundDesc {                  // device resident: the round's shape set
  int ns; int pad[3];
  int slot[RSMAX];
  Req reqs[RSMAX];
};

struct RoundCtl {                   // device resident: progress of the batch, written by the resolver
  int next_p, p_end, error, rounds;
  long long pods, tracked;
  long long stops[4];               // pod limit, shape outside the set, tracked table full, list dry
  long long prof[RPROF];
};

// One shard's candidate buffer (dynamic layout: shape capacity nsc, list depth rkm):
//   int len[nsc], more[nsc], fit[nsc]; u64 fd[nsc], sd[nsc]; cand[nsc][rkm] of cand_bytes each
// cand: key u64 @0 | rc[8] i32 @8 | rm[8] i32 @40 | mt i32 @72 | fterm u64 @80 | sbase u64 @88 |
//       sc[nsc] i32 @96 | al[nsc] u32 @96+4nsc | st[nsc] u8 @96+8nsc
struct BufLayout {
  int nsc, rkm, cand_bytes, pad;
  unsigned off_len, off_more, off_fit, off_fd, off_sd, off_cand;
  unsigned long long bytes;         // per shard, multiple of 16
};
static inline BufLayout make_layout(int ns, int rkm) {
  BufLayout L;
  L.nsc = (ns + 15) / 16 * 16; L.rkm = rkm; L.cand_bytes = 96 + 9 * L.nsc; L.pad = 0;
  unsigned o = 0;
  L.off_len = o; o += 4u * L.nsc;
  L.off_more = o; o += 4u * L.nsc;
  L.off_fit = o; o += 4u * L.nsc;
  o = (o + 15u) & ~15u;
  L.off_fd = o; o += 8u * L.nsc;
  L.off_sd = o; o += 8u * L.nsc;
  L.off_cand = o;
  L.bytes = (unsigned long long)o + (unsigned long long)L.nsc * rkm * L.cand_bytes;
  return L;
}
#define CD_KEY 0
#define CD_RC 8
#define CD_RM 40
#define CD_MT 72
#define CD_FT 80
#define CD_SB 88
#define CD_SC 96
#define CD_AL(nsc) (CD_SC + 4 * (nsc))
#define CD_ST(nsc) (CD_SC + 8 * (nsc))

// Read view of one candidate record (k_merge writes it).  Every reader goes through this view and cand_at.
struct Cand {
  const char *p; int nsc;
  __device__ __forceinline__ unsigned long long key() const { return *reinterpret_cast<const unsigned long long *>(p + CD_KEY); }
  __device__ __forceinline__ int row(int f) const { return reinterpret_cast<const int *>(p + CD_RC)[f]; }   // f < 16: rc[8], rm[8]
  __device__ __forceinline__ int mt() const { return *reinterpret_cast<const int *>(p + CD_MT); }
  __device__ __forceinline__ unsigned long long fterm() const { return *reinterpret_cast<const unsigned long long *>(p + CD_FT); }
  __device__ __forceinline__ unsigned long long sbase() const { return *reinterpret_cast<const unsigned long long *>(p + CD_SB); }
  __device__ __forceinline__ int sc(int s) const { return reinterpret_cast<const int *>(p + CD_SC)[s]; }
  __device__ __forceinline__ uint32_t al(int s) const { return reinterpret_cast<const uint32_t *>(p + CD_AL(nsc))[s]; }
  __device__ __forceinline__ uint8_t st(int s) const { return reinterpret_cast<const uint8_t *>(p + CD_ST(nsc))[s]; }
};
// entry k of the list of shape s in the candidate buffer of shard d
__device__ __forceinline__ Cand cand_at(const char *bufs, const BufLayout &L, int d, int s, int k) {
  return Cand{bufs + (size_t)d * L.bytes + L.off_cand + ((size_t)s * L.rkm + k) * L.cand_bytes, L.nsc};
}

struct AggPart { unsigned long long fd, sd; int fit, pad; };

struct TableSet {                   // all option tables of the handle
  uint8_t *st; int32_t *sc; uint8_t *al; size_t n_pad; int n_slots;
};
__device__ __forceinline__ uint8_t *tb_st(const TableSet &t, int slot) { return t.st + (size_t)slot * t.n_pad; }
__device__ __forceinline__ int32_t *tb_sc(const TableSet &t, int slot) { return t.sc + (size_t)slot * t.n_pad; }
__device__ __forceinline__ uint8_t *tb_al(const TableSet &t, int slot) { return t.al + (size_t)slot * EGS_C * t.n_pad; }

__device__ __forceinline__ bool ctl_idle(const RoundCtl *c) { return c && (c->next_p >= c->p_end || c->error != 0); }

struct SelectArgs {
  const int32_t *core, *mem, *mem_total;
  int lo, hi, policy, nsc;          // this shard's node range
  const RoundDesc *rd;
  TableSet tb;
  const uint8_t *obs_pending;       // per slot: shape observed since its OPT_NEW options were made
  unsigned long long *cta_lists;    // [grid][nsc][RK]
  AggPart *cta_agg;                 // [grid][nsc]
  const RoundCtl *ctl;              // batch finished -> nothing to do
};

// 32 keys, one per lane -> sorted descending across the lanes (bitonic network, 15 exchange steps)
__device__ __forceinline__ unsigned long long warp_sort_desc(unsigned long long v, int lane) {
#pragma unroll
  for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, v, j);
      const bool take_max = ((lane & j) == 0) == ((lane & k) == 0);
      v = take_max ? (o > v ? o : v) : (o < v ? o : v);
    }
  }
  return v;
}
// two descending lists (one key per lane each) -> the 32 largest of their union, descending:
// max(a[i], b[31-i]) is a bitonic sequence holding exactly those keys; 5 merge steps sort it
__device__ __forceinline__ unsigned long long merge_top32(unsigned long long a, unsigned long long b, int lane) {
  const unsigned long long br = __shfl_sync(0xffffffffu, b, 31 - lane);
  unsigned long long v = a > br ? a : br;
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) {
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, v, j);
    v = ((lane & j) == 0) ? (o > v ? o : v) : (o < v ? o : v);
  }
  return v;
}
// 128-key lists: element e = q*32 + lane lives in register q of lane `lane`, descending in e.
// A bitonic 128-sequence -> sorted descending (strides 64, 32 between registers; 16..1 by shuffle)
__device__ __forceinline__ void bitonic128_desc(unsigned long long (&A)[RQMAX], int lane) {
#pragma unroll
  for (int q = 0; q < 2; q++) { const unsigned long long x = A[q], y = A[q + 2]; A[q] = x > y ? x : y; A[q + 2] = x > y ? y : x; }
#pragma unroll
  for (int q = 0; q < 4; q += 2) { const unsigned long long x = A[q], y = A[q + 1]; A[q] = x > y ? x : y; A[q + 1] = x > y ? y : x; }
#pragma unroll
  for (int j = 16; j > 0; j >>= 1) {
#pragma unroll
    for (int q = 0; q < RQMAX; q++) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, A[q], j);
      A[q] = ((lane & j) == 0) ? (o > A[q] ? o : A[q]) : (o < A[q] ? o : A[q]);
    }
  }
}
// top 128 of (sorted 128-list A) U (sorted 32-list b)
__device__ __forceinline__ void merge32_into128(unsigned long long (&A)[RQMAX], unsigned long long b, int lane) {
  const unsigned long long kth = __shfl_sync(0xffffffffu, A[RQMAX - 1], 31);
  const unsigned long long bmax = __shfl_sync(0xffffffffu, b, 0);
  if (bmax <= kth) return;
  const unsigned long long br = __shfl_sync(0xffffffffu, b, 31 - lane);
  A[RQMAX - 1] = A[RQMAX - 1] > br ? A[RQMAX - 1] : br;
  bitonic128_desc(A, lane);
}
// top 128 of two sorted 128-lists
__device__ __forceinline__ void merge128(unsigned long long (&A)[RQMAX], const unsigned long long (&B)[RQMAX], int lane) {
#pragma unroll
  for (int q = 0; q < RQMAX; q++) {
    const unsigned long long br = __shfl_sync(0xffffffffu, B[RQMAX - 1 - q], 31 - lane);
    A[q] = A[q] > br ? A[q] : br;
  }
  bitonic128_desc(A, lane);
}

// --------------------------------------------------------------------------------------------
// k_select
// --------------------------------------------------------------------------------------------
// k_select_nodes (a batch under a node set): an excluded node is skipped whole -- no Trade, no NEW -> CACHED, no fit
// count, no digest, no list key -- so the candidate lists, and with them every node the resolver tracks, hold only
// admitted nodes.
template <bool MASKED>
__device__ __forceinline__ void select_body(const SelectArgs &a, NodeSet set) {
  __shared__ unsigned long long s_list[SEL_WARPS][32][RK];
  __shared__ AggPart s_agg[SEL_WARPS][32];
  __shared__ Req s_reqs[32];          // the round descriptor is indexed dynamically: stage it in smem
  __shared__ int s_slot[32];
  if (ctl_idle(a.ctl)) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gwarp = blockIdx.x * SEL_WARPS + warp, nwarps = gridDim.x * SEL_WARPS;
  const int ns = a.rd->ns;
  static_assert(RK == 32, "top-K lists are one key per lane");
  const int n_chunks = (a.hi - a.lo + 127) / 128;
  for (int g0 = 0; g0 < ns; g0 += 32) {                          // shape groups of 32
    const int gn = min(32, ns - g0);
    __syncthreads();
    if (threadIdx.x < gn) { s_slot[threadIdx.x] = a.rd->slot[g0 + threadIdx.x]; s_reqs[threadIdx.x] = a.rd->reqs[g0 + threadIdx.x]; }
    for (int s = lane; s < 32; s += 32) { s_agg[warp][s].fd = 0; s_agg[warp][s].sd = 0; s_agg[warp][s].fit = 0; }
    for (int i = lane; i < 32 * RK; i += 32) (&s_list[warp][0][0])[i] = 0;
    __syncthreads();
    for (int chunk = gwarp; chunk < n_chunks; chunk += nwarps) {
      const int base = a.lo + chunk * 128 + lane;               // lane handles nodes base + 32*j: tied scores arrive in key order
      unsigned long long h1[4], h2[4];                          // per-node digest hashes, shared by all shapes
#pragma unroll
      for (int j = 0; j < 4; j++) { h1[j] = fit_term((uint32_t)(base + 32 * j)); h2[j] = score_base((uint32_t)(base + 32 * j)); }
      for (int s = 0; s < gn; s++) {
        const int slot = s_slot[s];
        uint8_t *stp = tb_st(a.tb, slot);
        int32_t *scp = tb_sc(a.tb, slot);
        uint8_t *alp = tb_al(a.tb, slot);
        const bool pending = a.obs_pending[slot] != 0;
        const Req &r = s_reqs[s];
        const bool single = req_is_single(r);
        uint8_t st[4]; int sc[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int i = base + 32 * j;
          // an excluded node reads as a node past hi: OPT_UNFIT, which the loop below neither Trades, writes nor counts
          st[j] = i < a.hi && (!MASKED || set.admits(i)) ? stp[i] : (uint8_t)OPT_UNFIT;
          sc[j] = i < a.hi ? scp[i] : 0;
        }
        unsigned long long key[4], fd = 0, sd = 0;
        int fit = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const int i = base + 32 * j;
          key[j] = 0;
          if (i >= a.hi) continue;
          const uint8_t st0 = st[j];
          if (st[j] == OPT_NEW && pending) st[j] = OPT_CACHED;
          if (st[j] == OPT_ABSENT) {                             // full evaluate (gpu.go:65-129)
            int c[EGS_G], m[EGS_G]; uint32_t masks;
            load_row(a.core, a.mem, (size_t)i, c, m);
            if (trade_any(c, m, a.mem_total[i], r, single, a.policy, sc[j], masks)) {
              st[j] = OPT_NEW;
              scp[i] = sc[j];
              for (int k = 0; k < r.C; k++) alp[(size_t)k * a.tb.n_pad + i] = (uint8_t)(masks >> (8 * k));
            } else {
              st[j] = OPT_UNFIT;
            }
          }
          if (st[j] != st0) stp[i] = st[j];
          if (st[j] == OPT_CACHED || st[j] == OPT_NEW) {
            key[j] = cand_key(sc[j], (uint32_t)i);
            fit++; fd += h1[j]; sd += score_term_b(h2[j], sc[j]);
          }
        }
        fit = warp_sum_i32(fit); fd = warp_sum_u64(fd); sd = warp_sum_u64(sd);
        if (lane == 0) { s_agg[warp][s].fit += fit; s_agg[warp][s].fd += fd; s_agg[warp][s].sd += sd; }
        // top-32 of this warp for shape s: sort 32 keys, merge sorted lists
        unsigned long long L = s_list[warp][s][lane];
        bool changed = false;
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const unsigned long long kth = __shfl_sync(0xffffffffu, L, RK - 1);
          if (__ballot_sync(0xffffffffu, key[j] > kth)) { L = merge_top32(L, warp_sort_desc(key[j], lane), lane); changed = true; }
        }
        if (changed) s_list[warp][s][lane] = L;
        __syncwarp();
      }
    }
    __syncthreads();
    // fold the warps of this CTA: warp w owns shapes s == w (mod SEL_WARPS)
    for (int s = warp; s < gn; s += SEL_WARPS) {
      unsigned long long L = s_list[0][s][lane];
      for (int w = 1; w < SEL_WARPS; w++) L = merge_top32(L, s_list[w][s][lane], lane);
      a.cta_lists[((size_t)blockIdx.x * a.nsc + g0 + s) * RK + lane] = L;
      if (lane == 0) {
        AggPart t; t.fd = 0; t.sd = 0; t.fit = 0; t.pad = 0;
        for (int w = 0; w < SEL_WARPS; w++) { t.fd += s_agg[w][s].fd; t.sd += s_agg[w][s].sd; t.fit += s_agg[w][s].fit; }
        a.cta_agg[(size_t)blockIdx.x * a.nsc + g0 + s] = t;
      }
    }
  }
}
__global__ void __launch_bounds__(SEL_THREADS) k_select(SelectArgs a) { select_body<false>(a, NodeSet{nullptr}); }
__global__ void __launch_bounds__(SEL_THREADS) k_select_nodes(SelectArgs a, NodeSet set) { select_body<true>(a, set); }

// --------------------------------------------------------------------------------------------
// k_merge: one CTA per shape of the round
// --------------------------------------------------------------------------------------------
struct MergeArgs {
  const int32_t *core, *mem, *mem_total;
  const RoundDesc *rd;
  TableSet tb;
  uint8_t *obs_pending;
  const unsigned long long *cta_lists; const AggPart *cta_agg; int n_cta;
  char *out; BufLayout L;           // this shard's candidate buffer
  const RoundCtl *ctl;
};

__global__ void __launch_bounds__(256) k_merge(MergeArgs a) {
  __shared__ unsigned long long s_l[8][RQMAX * 32];
  __shared__ AggPart s_a[8];
  __shared__ unsigned long long s_floor[8];
  __shared__ unsigned long long s_final[RQMAX * 32];
  __shared__ int s_len;
  if (ctl_idle(a.ctl)) return;
  const int s = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ns = a.rd->ns, nsc = a.L.nsc;
  unsigned long long A[RQMAX] = {0, 0, 0, 0};
  unsigned long long floor_k = 0;    // the merged list is exact down to the largest LAST key of a full CTA list
  AggPart ag; ag.fd = 0; ag.sd = 0; ag.fit = 0; ag.pad = 0;
  for (int c = warp; c < a.n_cta; c += 8) {
    const unsigned long long b = a.cta_lists[((size_t)c * nsc + s) * RK + lane];
    const unsigned long long last = __shfl_sync(0xffffffffu, b, 31);
    floor_k = last > floor_k ? last : floor_k;
    merge32_into128(A, b, lane);
    if (lane == 0) { const AggPart p = a.cta_agg[(size_t)c * nsc + s]; ag.fd += p.fd; ag.sd += p.sd; ag.fit += p.fit; }
  }
#pragma unroll
  for (int q = 0; q < RQMAX; q++) s_l[warp][q * 32 + lane] = A[q];
  if (lane == 0) { s_a[warp] = ag; s_floor[warp] = floor_k; }
  __syncthreads();
  if (warp == 0) {
    for (int w = 1; w < 8; w++) {
      unsigned long long B[RQMAX];
#pragma unroll
      for (int q = 0; q < RQMAX; q++) B[q] = s_l[w][q * 32 + lane];
      merge128(A, B, lane);
      floor_k = s_floor[w] > floor_k ? s_floor[w] : floor_k;
    }
    int cnt = 0;
#pragma unroll
    for (int q = 0; q < RQMAX; q++) {
      s_final[q * 32 + lane] = A[q];
      cnt += __popc(__ballot_sync(0xffffffffu, A[q] != 0 && A[q] >= floor_k));
    }
    if (lane == 0) {
      AggPart t = s_a[0];
      for (int w = 1; w < 8; w++) { t.fd += s_a[w].fd; t.sd += s_a[w].sd; t.fit += s_a[w].fit; }
      const int len = cnt < a.L.rkm ? cnt : a.L.rkm;
      s_len = len;
      reinterpret_cast<int *>(a.out + a.L.off_len)[s] = len;
      reinterpret_cast<int *>(a.out + a.L.off_more)[s] = t.fit > len;
      reinterpret_cast<int *>(a.out + a.L.off_fit)[s] = t.fit;
      reinterpret_cast<unsigned long long *>(a.out + a.L.off_fd)[s] = t.fd;
      reinterpret_cast<unsigned long long *>(a.out + a.L.off_sd)[s] = t.sd;
      a.obs_pending[a.rd->slot[s]] = 0;                        // consumed by this round's select
    }
  }
  __syncthreads();
  // payload: 16 threads per candidate, 16 candidates per pass
  const int len = s_len;
  for (int k = threadIdx.x >> 4; k < a.L.rkm; k += 16) {
    const int f = threadIdx.x & 15;
    char *cd = a.out + a.L.off_cand + ((size_t)s * a.L.rkm + k) * a.L.cand_bytes;
    if (k >= len) { if (f == 0) *reinterpret_cast<unsigned long long *>(cd + CD_KEY) = 0; continue; }
    const unsigned long long key = s_final[k];
    const size_t node = key_node(key);
    if (f == 0) { *reinterpret_cast<unsigned long long *>(cd + CD_KEY) = key; *reinterpret_cast<int *>(cd + CD_MT) = a.mem_total[node]; *reinterpret_cast<int *>(cd + CD_MT + 4) = 0; }
    if (f == 1) *reinterpret_cast<unsigned long long *>(cd + CD_FT) = fit_term((uint32_t)node);
    if (f == 2) *reinterpret_cast<unsigned long long *>(cd + CD_SB) = score_base((uint32_t)node);
    if (f < EGS_G) reinterpret_cast<int *>(cd + CD_RC)[f] = a.core[node * EGS_G + f];
    else reinterpret_cast<int *>(cd + CD_RM)[f - EGS_G] = a.mem[node * EGS_G + f - EGS_G];
    int *csc = reinterpret_cast<int *>(cd + CD_SC);
    uint32_t *cal = reinterpret_cast<uint32_t *>(cd + CD_AL(nsc));
    uint8_t *cst = reinterpret_cast<uint8_t *>(cd + CD_ST(nsc));
    for (int s2 = f; s2 < nsc; s2 += 16) {
      uint8_t st = OPT_UNFIT; int32_t sc = 0; uint32_t al = 0;
      if (s2 < ns) {
        const int slot = a.rd->slot[s2];
        st = tb_st(a.tb, slot)[node]; sc = tb_sc(a.tb, slot)[node];
        const uint8_t *alp = tb_al(a.tb, slot);
        for (int c = 0; c < EGS_C; c++) al |= (uint32_t)alp[(size_t)c * a.tb.n_pad + node] << (8 * c);
      }
      cst[s2] = st; csc[s2] = sc; cal[s2] = al;
    }
  }
}

// --------------------------------------------------------------------------------------------
// k_resolve_mw: one CTA, one owner warp per shape (shape index si is owned by warp si % nw)
// --------------------------------------------------------------------------------------------
#ifdef EGS_RESOLVE_PROF
#define PROF_T(i) { long long now_ = clock64(); prof[i] += now_ - tprev; tprev = now_; }
#define PROF_C(i, v) { prof[i] += (v); }
#define PROF_RELEASE() { *reinterpret_cast<volatile long long *>(&S.t_release) = clock64(); }   // lane 0, before the arrive
#else
#define PROF_T(i)
#define PROF_C(i, v)
#define PROF_RELEASE()
#endif

// max of a 64-bit key over the warp: two redux.sync steps on the halves; owner = lowest lane holding it
__device__ __forceinline__ unsigned long long warp_max_key_fwd(unsigned long long mine, int &owner_lane) {
  const unsigned hi = (unsigned)(mine >> 32);
  const unsigned m1 = __reduce_max_sync(0xffffffffu, hi);
  const unsigned m2 = __reduce_max_sync(0xffffffffu, hi == m1 ? (unsigned)mine : 0u);
  const unsigned long long win = ((unsigned long long)m1 << 32) | m2;
  owner_lane = __ffs(__ballot_sync(0xffffffffu, mine == win)) - 1;
  return win;
}

struct MwArgs {
  int32_t *core, *mem;              // write-back targets
  int lo, hi, policy, n_shards;
  const RoundDesc *rd;
  TableSet tb;
  uint8_t *obs_pending;
  const char *bufs; BufLayout L;    // [n_shards] candidate buffers
  const uint8_t *pod_sidx;          // per pod: index of its shape in the round set
  int p0, p_limit;                  // p0 < 0: pods [ctl->next_p, ctl->p_end)
  PodOut out;
  RoundCtl *ctl;
  int rke;                          // list entries per (shape, shard) held in shared memory
  int nw;                           // worker warps
  int pre_h, pre_cap;               // pre-install: the first pre_h merged candidates of every shape, at most pre_cap slots
};

template <int NS, int NT>
struct MwSmem {
  static constexpr int HS = 2 * NT;                        // open-addressed set of tracked node ids
  // ---- owner-private per shape (only the owner warp of shape s touches row s; slots >= the owner's view of nT
  //      are written by the warp that installs them, inside its ticket)
  unsigned long long tkey[NS][NT];   // cand_key of a tracked node's option when it is fit (CACHED/NEW), else 0
  unsigned long long hkey[NS][RD];   // current head of each untracked list (0 = none); may be STALE (see maintain_heads)
  unsigned long long afd[NS], asd[NS], bh[NS];             // aggregates; best head over the shards
  unsigned long long dbound[NS];     // largest LAST key of an exhausted truncated list: unseen nodes stay below it (0: none)
  unsigned long long xbest[NS];      // best key among slots OTHER shapes installed since the owner's last ticket
  uint32_t al[NS][NT];               // option.Allocated masks
  unsigned pmask[NS][NT / 32];       // tracked slots whose option is ABSENT: Trade at the shape's next pod
  int afit[NS], bh_d[NS], observed[NS], xbest_t[NS], hv_nT[NS], hpay_node[NS];
  int pu[NS];                        // summary of pmask[s]: -1 none, t >= 0 exactly slot t, -2 unknown / several
  int rq_single[NS], rq_core[NS], rq_mem[NS]; uint32_t rq_cmask[NS];
  uint8_t st[NS][NT];                // OPT_*
  uint8_t cur[NS][RD], len[NS][RD], more[NS][RD];
  Req reqs[NS];
  // ---- shared, changed only inside a ticket
  unsigned long long fterm[NT], sbase[NT];                 // fit_term / score_base of each tracked slot's node
  int node[NT], mt[NT], dirty[NT];
  int ver[NT];                       // seqlock of the slot's rows: odd while a bind is writing them, +2 per bind
  int rc[NT][EGS_G], rm[NT][EGS_G];
  int hset[HS];
  unsigned long long mbar[MW_MAX_WARPS];   // one per owner warp: "the ticket is yours"
  int turn;                                // the pod whose ticket is open; MW_STOP | p once the round was stopped before pod p
  int stop, stop_reason, stop_p, nT, n_observed, mono, p0, p_end;
#ifdef EGS_RESOLVE_PROF
  long long t_release;                     // clock64 at which the last ticket was handed on
#endif
};
#define MW_STOP 0x40000000

// The resolver instances, by the size of the round's shape set: NS shapes, NT tracked slots, lists of RKM merged
// candidates per shape and shard.  kHpay: shared memory holds one prefetched candidate payload per shape (cp.async).
// kPreinstall: the prologue pre-installs the round's likely winners (DESIGN §3.1).  Neither is in the 96-shape /
// 128-slot resolver: there (config 3: multi-container shapes, nearly every pod a general pod whose in-ticket scans grow
// with the number of slots) pre-install measured slower.
template <int NS_, int NT_, int RKM_, bool PRE_, bool HPAY_>
struct MwInst {
  static constexpr int NS = NS_, NT = NT_, RKM = RKM_;
  static constexpr bool kPreinstall = PRE_, kHpay = HPAY_;
  using Smem = MwSmem<NS, NT>;
};
using MwInst16 = MwInst<16, 512, 128, true, true>;
using MwInst32 = MwInst<32, 256, 64, true, true>;
using MwInst96 = MwInst<RSMAX, 128, 32, false, false>;

// Dynamic shared memory of instance I: MwSmem, then the tail -- the lists lk (u64 [ns][D][rke]), the prefetched
// payloads hpay (kHpay: [ns][cand_bytes]) and psrc (kPreinstall: int[NT], the candidate entry each pre-installed slot
// comes from).  Byte offsets; `end` is the size.
struct MwTail { size_t lk, hpay, psrc, end; };
template <class I>
__host__ __device__ __forceinline__ MwTail mw_tail(int ns, int D, int rke, int cand_bytes) {
  MwTail t;
  t.lk = (sizeof(typename I::Smem) + 15) & ~(size_t)15;
  t.hpay = t.lk + (size_t)ns * D * rke * 8;
  t.psrc = t.hpay + (I::kHpay ? (size_t)ns * cand_bytes : 0);
  t.end = t.psrc + (I::kPreinstall ? sizeof(int) * I::NT : 0);
  return t;
}

// ---- the resolver instance for a round set of ns shapes: f(MwInst16()), f(MwInst32()) or f(MwInst96())
template <class F>
static auto mw_dispatch(int ns, F &&f) {
  if (ns <= MwInst16::NS) return f(MwInst16());
  if (ns <= MwInst32::NS) return f(MwInst32());
  return f(MwInst96());
}
#define MW_SMEM_MAX 232448   // 227 KB opt-in limit per CTA on sm_90

// Pre-install (DESIGN §3.1): the resolver's prologue fills 3/4 of the tracked table with the top NT / ns merged
// candidates of every shape (at most half of a list held in shared memory, so no list runs dry at once); the last
// quarter stays free for first pods and new winners.  Only in the instances with kPreinstall.
template <class I>
static void preinstall_geometry(int ns, int rke, int &h, int &cap) {
  h = 0; cap = 0;
  if (!I::kPreinstall) return;
  h = std::max(1, std::min(I::NT / std::max(ns, 1), rke / 2));
  cap = 3 * I::NT / 4;
}

// Geometry of the resolver for a round set of ns shapes (1..RSMAX) over D shards:
//   rkm      list depth k_merge gathers per (shape, shard) -- the instance's RKM, at most 64 above two shards: every
//            shard contributes its own list, so the resolver holds about as many candidates per shape in total
//   rke      list entries per (shape, shard) the resolver keeps in shared memory: rkm, or what fits next to MwSmem
//            (even, so that what follows the lists stays 16-byte aligned); below rkm a list is truncated (`more`)
//   smem     dynamic shared memory of k_resolve_mw
//   pre_h, pre_cap   pre-install (preinstall_geometry)
// batch_rounds refuses a set with rke < 4.  Pure host arithmetic.
struct MwGeometry { int rkm, rke, pre_h, pre_cap; size_t smem; };
static inline MwGeometry mw_geometry(int ns, int D) {
  MwGeometry g;
  g.rkm = mw_dispatch(ns, [](auto i) { return decltype(i)::RKM; });
  if (D > 2) g.rkm = std::min(g.rkm, 64);
  const int cand_bytes = make_layout(ns, g.rkm).cand_bytes;
  g.rke = g.rkm;
  mw_dispatch(ns, [&](auto i) {
    using I = decltype(i);
    const size_t avail = MW_SMEM_MAX - mw_tail<I>(ns, D, 0, cand_bytes).end;   // all but the lists
    const size_t per = (size_t)ns * D * 8;
    if ((size_t)g.rke * per > avail) g.rke = (int)(avail / per) & ~1;
    g.smem = mw_tail<I>(ns, D, g.rke, cand_bytes).end;
    preinstall_geometry<I>(ns, g.rke, g.pre_h, g.pre_cap);
  });
  return g;
}

// Ticket hand-over: `turn` in shared memory names the pod whose ticket is open (bookkeeping, and the stop signal);
// the owner of the next pod SLEEPS in hardware on its own mbarrier (try_wait suspends the warp) and is woken by ONE
// arrive of the warp that finished the previous pod.  Alternatives (tools/micro/handoff_bench.cu measures the bare
// hand-over): every warp polling one word steals issue slots from the ticket holder, and a two-level scheme (only the
// next owners poll, the others sleep) was slower than this; a bare hand-over costs about the same whatever the
// mechanism.
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {   // release.cta
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, unsigned parity) {   // acquire.cta
  unsigned ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"((unsigned)__cvta_generic_to_shared(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ int ld_vol(const int *p) { return *reinterpret_cast<const volatile int *>(p); }
__device__ __forceinline__ void st_vol(int *p, int v) { *reinterpret_cast<volatile int *>(p) = v; }

template <class SM>
__device__ __forceinline__ unsigned hset_slot(uint32_t node) {
  return ((node * 2654435761u) >> 8) & (unsigned)(SM::HS - 1);
}
template <class SM>
__device__ __forceinline__ bool hset_has(const SM &S, uint32_t node) {
  for (unsigned i = hset_slot<SM>(node);; i = (i + 1) & (unsigned)(SM::HS - 1)) {
    const int v = ld_vol(&S.hset[i]);
    if (v == (int)node) return true;
    if (v < 0) return false;
  }
}
template <class SM>
__device__ __forceinline__ void hset_add(SM &S, uint32_t node) {   // one lane, inside a ticket; at most NT entries (load <= 1/2)
  unsigned i = hset_slot<SM>(node);
  while (S.hset[i] >= 0) i = (i + 1) & (unsigned)(SM::HS - 1);
  st_vol(&S.hset[i], (int)node);
}
template <class SM>
__device__ __forceinline__ void hset_add_concurrent(SM &S, uint32_t node) {   // several lanes at once, distinct nodes
  unsigned i = hset_slot<SM>(node);
  while (atomicCAS(&S.hset[i], -1, (int)node) != -1) i = (i + 1) & (unsigned)(SM::HS - 1);
}

// The untracked candidate lists of shape s belong to its owner warp and are maintained LAZILY, outside the ticket:
// entries whose node is tracked by now are skipped.  A head may therefore be STALE (its node became tracked after
// this ran).  What the ticket may rely on, whatever the timing of this maintenance:
//   * U = max(bh[s], dbound[s]) is an UPPER BOUND of the key of every untracked candidate of the shape: a list is
//     sorted, so its (possibly stale) head bounds its later entries and -- when truncated -- the unseen nodes; an
//     exhausted truncated list is bounded by its last key (dbound).  best tracked >= U  =>  a tracked option wins.
//   * otherwise the ticket re-runs this maintenance INSIDE the ordered section (force), where the tracked set is
//     exact, and decides on exact heads.  Every decision -- in particular where a round stops -- is thus a function
//     of the serial state only, never of timing: the replicated resolvers of a sharded run stay in lock step.
// Lanes d < D work on list (s, d).
template <class SM>
__device__ __forceinline__ void maintain_heads(SM &S, const unsigned long long *lk, int D, int rke, int s, int lane, bool force) {
  const int nT = ld_vol(&S.nT);
  if (!force && S.hv_nT[s] == nT) return;                       // no node became tracked since the last look
  unsigned long long k = 0, db = 0;
  if (lane < D) {
    const int d = lane;
    int c = S.cur[s][d];
    const int len = S.len[s][d];
    const unsigned long long *l = lk + ((size_t)s * D + d) * rke;
    while (c < len) { k = l[c]; if (!hset_has(S, key_node(k))) break; c++; }
    if (c >= len) { k = 0; if (S.more[s][d] != 0 && len > 0) db = l[len - 1]; }
    S.cur[s][d] = (uint8_t)c;
    S.hkey[s][d] = k;
  }
  if (D == 1) {                                                  // one list (unsharded): lane 0 holds the maxima already
    if (lane == 0) { S.bh[s] = k; S.bh_d[s] = 0; S.dbound[s] = db; S.hv_nT[s] = nT; }
    __syncwarp();
    return;
  }
  int owner, o2;
  const unsigned long long b = warp_max_key_fwd(k, owner);
  const unsigned long long dbm = warp_max_key_fwd(db, o2);
  if (lane == 0) { S.bh[s] = b; S.bh_d[s] = b ? owner : 0; S.dbound[s] = dbm; S.hv_nT[s] = nT; }
  __syncwarp();
}

// Trade of one fractional single-container request on a tracked node, one lane per GPU (lane & 7), every
// lane holding the whole row: no shuffles until the final max.  Returns the folded key q*8+g (-1: no fit).
__device__ __forceinline__ int trade_lanes(const int (&c)[EGS_G], const int (&m)[EGS_G], int gl, int rq_c, int rq_m, int policy) {
  return __reduce_max_sync(0xffffffffu, trade_lane_key(c, m, gl, rq_c, rq_m, policy));
}

// ---- installing a tracked slot from its candidate record, in two parts shared by the ticket (install_slot, one warp)
// and the prologue (preinstall_slots, the whole CTA).  The caller sets node[t] and enters the node in the tracked set.
// Part f < 16 of the rows of slot t: rc[f] or rm[f - 8]; part 0 also writes the per-slot fields.
template <class SM>
__device__ __forceinline__ void install_rows(SM &S, const Cand &c, int t, int f) {
  const int v = c.row(f);
  if (f < EGS_G) S.rc[t][f] = v; else S.rm[t][f - EGS_G] = v;
  if (f == 0) { S.mt[t] = c.mt(); S.dirty[t] = 0; S.ver[t] = 0; S.fterm[t] = c.fterm(); S.sbase[t] = c.sbase(); }
}
// The option of shape s2 on slot t (node w); an OPT_NEW option of an observed shape is an ordinary cached one.
// Returns its key (0: not fit).
template <class SM>
__device__ __forceinline__ unsigned long long install_option(SM &S, const Cand &c, int t, uint32_t w, int s2, bool observed) {
  uint8_t st = c.st(s2);
  if (st == OPT_NEW && observed) st = OPT_CACHED;
  const unsigned long long k = (st == OPT_CACHED || st == OPT_NEW) ? cand_key(c.sc(s2), w) : 0ull;
  S.st[s2][t] = st; S.al[s2][t] = c.al(s2); S.tkey[s2][t] = k;
  if (st == OPT_ABSENT) { atomicOr(&S.pmask[s2][t >> 5], 1u << (t & 31)); S.pu[s2] = -2; }   // select leaves none; kept for safety
  return k;
}

// A node becomes tracked: install the record `c` (node w) as slot t.  All lanes, inside the ticket of shape s_self.
// Other shapes learn about the slot through xbest (their owners scan only the slots they have seen).
template <class SM>
__device__ __noinline__ void install_slot(SM &S, Cand c, int t, uint32_t w, int ns, int s_self, int lane) {
  if (lane < 2 * EGS_G) {
    install_rows(S, c, t, lane);
    if (lane == 0) { S.node[t] = (int)w; hset_add(S, w); }
  }
  for (int s2 = lane; s2 < ns; s2 += 32) {
    const unsigned long long k = install_option(S, c, t, w, s2, S.observed[s2] != 0);
    if (s2 != s_self && k > S.xbest[s2]) { S.xbest[s2] = k; S.xbest_t[s2] = t; }
  }
}

// record of the current best head of shape s: prefetched copy in shared memory, else the candidate buffer
template <class SM>
__device__ __forceinline__ Cand head_payload(const SM &S, const MwArgs &a, const char *hpay, int s, uint32_t w) {
  if (hpay && S.hpay_node[s] == (int)w) return Cand{hpay + (size_t)s * a.L.cand_bytes, a.L.nsc};
  const int d = S.bh_d[s];
  return cand_at(a.bufs, a.L, d, s, S.cur[s][d]);
}

// Single-container Transact (gpu.go:164-171) of GPU g of tracked slot t, all lanes, inside the ticket: the row is
// written under the slot's seqlock.  Returns ok (the bind is recorded -- dirty -- either way).
template <class SM>
__device__ __forceinline__ int bind_single_slot(SM &S, int t, int g, int rq_c, int rq_m, int lane) {
  const int c = S.rc[t][g], m = S.rm[t][g];
  const int ok = (c >= rq_c && m >= rq_m) ? 1 : 0;
  __syncwarp();                                                  // every lane has read the row
  if (lane == 0) {
    if (ok) { const int v = S.ver[t]; st_vol(&S.ver[t], v + 1); S.rc[t][g] = c - rq_c; S.rm[t][g] = m - rq_m; st_vol(&S.ver[t], v + 2); }
    S.dirty[t] = 1;
  }
  return ok;
}

// node.go:90-92: the winning option (key win, slot t) of shape s is consumed; the aggregates (fit, fd, sd as this pod
// saw them) lose its terms, and it is the shape's one pending option.  One lane.
template <class SM>
__device__ __forceinline__ void consume_option(SM &S, int s, int t, unsigned long long win, int fit, unsigned long long fd,
                                               unsigned long long sd) {
  S.st[s][t] = OPT_ABSENT; S.tkey[s][t] = 0; S.pmask[s][t >> 5] |= 1u << (t & 31);
  S.afit[s] = fit - 1; S.afd[s] = fd - S.fterm[t]; S.asd[s] = sd - score_term_b(S.sbase[t], key_score(win));
  S.pu[s] = t;
}

// General Trade of request r on the tracked slot whose rows are (rc, rm): the DFS leaves spread over the lanes
// (trade_leaf_eval), the winner = maximal (score, leaf index).  Warp-uniform result.
__device__ __forceinline__ bool trade_warp(const int *rc, const int *rm, int mem_total, const Req &r, int policy, int lane,
                                           int &score, uint32_t &masks) {
  int c[EGS_G], m[EGS_G];
#pragma unroll
  for (int g = 0; g < EGS_G; g++) { c[g] = rc[g]; m[g] = rm[g]; }
  int bits, nbranch, nleaf;
  trade_leaf_space(c, r, bits, nbranch, nleaf);
  unsigned long long best = 0;                                   // ((score << 32) | leaf) + 1; 0 = no feasible leaf
  for (int leaf = lane; leaf < nleaf; leaf += 32) {
    uint32_t mk;
    const int sc = trade_leaf_eval(c, m, mem_total, r, policy, bits, nbranch, leaf, mk);
    if (sc >= 0) { const unsigned long long k = (((unsigned long long)(unsigned)sc << 32) | (unsigned)leaf) + 1ull; best = k > best ? k : best; }
  }
  int owner;
  const unsigned long long win = warp_max_key_fwd(best, owner);
  if (win == 0) return false;
  const int leaf = (int)(unsigned)(win - 1ull);
  score = trade_leaf_eval(c, m, mem_total, r, policy, bits, nbranch, leaf, masks);   // every lane: the winner's masks
  return true;
}

// ---- general pod (inside the ticket, whole warp): any shape, any number of pending options, any regime.
// Returns 0, or the stop reason (nothing was changed for this pod then).
template <class SM>
__device__ __noinline__ int general_pod(SM &S, const MwArgs &a, const unsigned long long *lk, const char *hpay, int lane, int p, int s, int ns) {
  const int grp = lane >> 3, gl = lane & 7;
  const unsigned gmask = 0xFFu << (8 * grp);
  const bool mono = S.mono != 0;
  int nT = S.nT;
  if (nT >= SM::HS / 2) return 2;                               // no free tracked slot for a new winner
  maintain_heads(S, lk, a.n_shards, a.rke, s, lane, true);      // inside the ticket the tracked set is exact
  if (lane == 0) { S.xbest[s] = 0; S.xbest_t[s] = -1; }         // the scan below sees every slot
  if (!S.observed[s]) {                                         // first pod of this shape in the round:
    for (int t = lane; t < nT; t += 32) if (S.st[s][t] == OPT_NEW) S.st[s][t] = OPT_CACHED;   // NEW options are now ordinary
    __syncwarp();
    if (lane == 0) { S.observed[s] = 1; S.n_observed = S.n_observed + 1; }
    __syncwarp();
  }
  const int single = S.rq_single[s];
  // tracked nodes: Trade absent options NOW (this pod's filter); best tracked option
  unsigned long long best = 0; int best_t = -1;
  const int nwords = (nT + 31) >> 5;
  for (int w = 0; w < nwords; w++) {
    unsigned word = S.pmask[s][w];
    if (word) {
      if (single) {
        // 8 lanes per pending node (lane == GPU), up to 4 nodes at a time
        const int rq_c = S.rq_core[s], rq_m = S.rq_mem[s];
        while (word) {
          int bsel = -1;
#pragma unroll
          for (int q = 0; q < 4; q++) {
            const int b = word ? __ffs(word) - 1 : -1;
            if (word) word &= word - 1;
            if (q == grp) bsel = b;
          }
          bool okl = false; int sc = 0; int t = 0;
          if (bsel >= 0) {                                       // group-uniform
            t = w * 32 + bsel;
            const int4 c0 = *reinterpret_cast<const int4 *>(&S.rc[t][0]), c1 = *reinterpret_cast<const int4 *>(&S.rc[t][4]);
            const int4 m0 = *reinterpret_cast<const int4 *>(&S.rm[t][0]), m1 = *reinterpret_cast<const int4 *>(&S.rm[t][4]);
            const int c[EGS_G] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
            const int m[EGS_G] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
            const int bk = __reduce_max_sync(gmask, trade_lane_key(c, m, gl, rq_c, rq_m, a.policy));
            if (gl == 0) {
              if (bk >= 0) {
                sc = a.policy == EGS_BINPACK ? (bk >> 3) * 100 : 0;
                S.st[s][t] = OPT_CACHED; S.al[s][t] = 1u << (bk & 7); S.tkey[s][t] = cand_key(sc, (uint32_t)S.node[t]);
                okl = true;
              } else {
                S.st[s][t] = OPT_UNFIT;
              }
            }
          }
          for (unsigned rem = __ballot_sync(0xffffffffu, okl); rem; rem &= rem - 1) {   // usually one leader
            if (lane == __ffs(rem) - 1) { S.afit[s] += 1; S.afd[s] += S.fterm[t]; S.asd[s] += score_term_b(S.sbase[t], sc); }
            __syncwarp();
          }
        }
      } else {
        for (unsigned rem = word; rem; rem &= rem - 1) {           // one pending node after the other, its DFS leaves over the lanes
          const int t = w * 32 + __ffs(rem) - 1;
          int sc = 0; uint32_t masks = 0;
          const bool ok = trade_warp(S.rc[t], S.rm[t], S.mt[t], S.reqs[s], a.policy, lane, sc, masks);
          if (lane == 0) {
            if (ok) {
              S.st[s][t] = OPT_CACHED; S.al[s][t] = masks; S.tkey[s][t] = cand_key(sc, (uint32_t)S.node[t]);
              S.afit[s] += 1; S.afd[s] += S.fterm[t]; S.asd[s] += score_term_b(S.sbase[t], sc);
            } else {
              S.st[s][t] = OPT_UNFIT;
            }
          }
          __syncwarp();
        }
      }
      __syncwarp();
      if (lane == 0) S.pmask[s][w] = 0;
    }
    const int t = w * 32 + lane;
    const unsigned long long k = t < nT ? S.tkey[s][t] : 0ull;
    if (k > best) { best = k; best_t = t; }
  }
  __syncwarp();
  // winner = max over (tracked options, best untracked list head); a stale head never exceeds the tracked maximum
  int owner;
  const unsigned long long tbest = warp_max_key_fwd(best, owner);
  const int tw0 = __shfl_sync(0xffffffffu, best_t, owner);
  const unsigned long long head = S.bh[s];
  const bool from_head = head > tbest;
  const unsigned long long win = from_head ? head : tbest;
  // a truncated list ran dry and what it did not show could beat the winner: the round must end (exact: the heads were
  // re-validated inside this ticket).  NOTE: the pending options Traded above stay Traded -- that is what the next
  // round's first filter of this shape would do on the same rows.
  if (S.dbound[s] > win) return 3;
  const int fitc = S.afit[s];
  const unsigned long long ofd = S.afd[s], osd = S.asd[s];
  // ---- commit: NodeAllocator.Allocate (node.go:87-104) on the tracked copy, or NOFIT
  int o_node = -1, o_status = EGS_ERR_NOFIT; uint32_t o_masks = 0;
  if (win != 0) {
    int t = tw0;
    if (from_head) {
      // an untracked node wins: it becomes tracked
      t = nT;
      const uint32_t w = key_node(win);
      asm volatile("cp.async.wait_all;" ::: "memory");
      __syncwarp();
      install_slot(S, head_payload(S, a, hpay, s, w), t, w, ns, s, lane);
      __syncwarp();
      nT = t + 1;
      if (lane == 0) { __threadfence_block(); st_vol(&S.nT, nT); }
      __syncwarp();
    }
    o_node = S.node[t];
    const uint32_t masks = S.al[s][t] & S.rq_cmask[s];
    const unsigned pbit = 1u << (t & 31);
    // NodeAllocator.Allocate: Transact, then the deferred delete of the option (node.go:90-92)
    int ok = 0;
    if (single) {
      ok = bind_single_slot(S, t, __ffs(masks) - 1, S.rq_core[s], S.rq_mem[s], lane);
      if (lane == 0) consume_option(S, s, t, win, fitc, ofd, osd);
    } else {
      __syncwarp();
      if (lane == 0) {
        consume_option(S, s, t, win, fitc, ofd, osd);
        S.dirty[t] = 1;
        const int v = S.ver[t]; st_vol(&S.ver[t], v + 1);
        ok = transact_row<EGS_G>(S.rc[t], S.rm[t], S.mt[t], S.reqs[s], masks) ? 1 : 0;
        st_vol(&S.ver[t], v + 2);
      }
      ok = __shfl_sync(0xffffffffu, ok, 0);
    }
    // Rows changed.  (a) not-yet-observed NEW options of this node are void (only while some shape of the
    // round is unobserved); (b) UNFIT memos are void -- unless the round is monotone (every container
    // fractional, every request >= 0; resolve_prologue): rows then only decrease and a fractional option
    // that did not fit can never fit (exact shortcut).
    if (!mono || S.n_observed < ns) {
      for (int s2 = lane; s2 < ns; s2 += 32) {
        if (s2 == s) continue;
        const uint8_t v = S.st[s2][t];
        if (v == OPT_UNFIT && !mono) { S.st[s2][t] = OPT_ABSENT; S.pmask[s2][t >> 5] |= pbit; S.pu[s2] = -2; }
        else if (v == OPT_NEW && !S.observed[s2]) {
          const unsigned long long k2 = S.tkey[s2][t];
          S.st[s2][t] = OPT_ABSENT; S.tkey[s2][t] = 0; S.pmask[s2][t >> 5] |= pbit; S.pu[s2] = -2;
          S.afit[s2] -= 1; S.afd[s2] -= S.fterm[t]; S.asd[s2] -= score_term_b(S.sbase[t], key_score(k2));
          if (S.xbest_t[s2] == t) { S.xbest[s2] = 0; S.xbest_t[s2] = -1; }   // (an unobserved shape rescans anyway)
        }
      }
    }
    __syncwarp();
    o_status = ok ? EGS_OK : EGS_ERR_TRANSACT;
    o_masks = ok ? masks : 0;
  }
  if (lane == 0) {
    if (win == 0) S.pu[s] = -1;                                 // every pending option of s was Traded above
    write_pod_out<EGS_G>(a.out, p, o_node, o_status, fitc, ofd, osd, o_masks);
  }
  __syncwarp();
  return 0;
}

// ---- pre-install (DESIGN §3.1).  The winner rule max(best tracked option, best untracked head) does not depend on
// WHICH nodes are tracked, so the prologue may track the round's likely winners before the first pod: their installs
// then leave the ordered section.  Selection (one warp): rank r = 0..pre_h-1, shape s = 0..ns-1 in that order, the
// entry of merged rank r of shape s over its D shard lists (a D-way merge on the lists' cursors), skipping nodes
// already chosen, until pre_cap slots.  Slot numbers follow that order: a function of the lists only, so the
// replicated resolvers of a sharded run make the same choice.  Returns the number of slots chosen.
template <class SM>
__device__ __noinline__ int preinstall_select(SM &S, const MwArgs &a, const unsigned long long *lk, int *psrc, int ns, int lane) {
  const int D = a.n_shards, rke = a.rke, H = a.pre_h, cap = a.pre_cap;
  int n = 0;
  for (int r = 0; r < H && n < cap; r++) {
    for (int g = 0; g < ns && n < cap; g += 32) {
      const int s = g + lane;
      int node = -1, src = 0;
      if (s < ns) {
        unsigned long long best = 0; int bd = 0, bc = 0;
        for (int d = 0; d < D; d++) {
          const int c = S.cur[s][d];
          const unsigned long long k = c < S.len[s][d] ? lk[((size_t)s * D + d) * rke + c] : 0ull;
          if (k > best) { best = k; bd = d; bc = c; }
        }
        if (best != 0) { S.cur[s][bd] = (uint8_t)(bc + 1); node = (int)key_node(best); src = (bd << 16) | (s << 8) | bc; }
      }
      bool take = node >= 0 && !hset_has(S, (uint32_t)node);
      const unsigned same = __match_any_sync(0xffffffffu, take ? node : -1 - lane);
      take = take && __ffs(same) - 1 == lane;                   // the lowest lane of a node chosen twice in this step
      const unsigned tm = __ballot_sync(0xffffffffu, take);
      const int t = n + __popc(tm & ((1u << lane) - 1u));
      if (take && t < cap) { S.node[t] = node; psrc[t] = src; hset_add_concurrent(S, (uint32_t)node); }
      n = min(cap, n + __popc(tm));
      __syncwarp();
    }
  }
  return n;
}

// Installs slots [0, nT) from their candidate entries (psrc: shard << 16 | shape << 8 | list position), all threads.
// install_slot without the ticket's parts: no xbest (every owner scans all slots at its first pod) and no shape is
// observed yet, so OPT_NEW stays NEW (the first pod of each shape turns it into CACHED).
template <class SM>
__device__ __noinline__ void preinstall_slots(SM &S, const MwArgs &a, const int *psrc, int nT, int ns) {
  const int tid = threadIdx.x, nthreads = blockDim.x;
  auto cand = [&](int t) { const int v = psrc[t]; return cand_at(a.bufs, a.L, v >> 16, (v >> 8) & 0xFF, v & 0xFF); };
  for (int i = tid; i < nT * 2 * EGS_G; i += nthreads) install_rows(S, cand(i / (2 * EGS_G)), i / (2 * EGS_G), i % (2 * EGS_G));
  for (int i = tid; i < nT * ns; i += nthreads) {
    const int t = i / ns, s2 = i - t * ns;
    install_option(S, cand(t), t, (uint32_t)S.node[t], s2, false);
  }
}

// ---- shared by the resolver kernels: round prologue (returns false when the batch is finished) and epilogue
template <class I>
__device__ __noinline__ bool resolve_prologue(typename I::Smem &S, const MwArgs &a, unsigned long long *lk, int *psrc, int &n_pre) {
  using SM = typename I::Smem;
  constexpr int NS = I::NS, NT = I::NT;
  const int tid = threadIdx.x, nthreads = blockDim.x;
  const int D = a.n_shards, rke = a.rke;
  const int ns = a.rd->ns;
  // ---- prologue
  {
    int p0 = a.p0, p_end = a.p_limit;
    if (a.p0 < 0) { if (ctl_idle(a.ctl)) return false; p0 = a.ctl->next_p; p_end = a.ctl->p_end; }
    if (tid == 0) { S.p0 = p0; S.p_end = p_end; S.turn = p0; S.stop = 0; S.stop_reason = 0; S.stop_p = p_end; S.nT = 0; S.n_observed = 0; }
    if (tid < MW_MAX_WARPS) mbar_init(&S.mbar[tid], 1);
  }
  for (int i = tid; i < SM::HS; i += nthreads) S.hset[i] = -1;
  for (int i = tid; i < NS * (NT / 32); i += nthreads) (&S.pmask[0][0])[i] = 0;
  for (int s = tid; s < NS; s += nthreads) {
    int fit = 0; unsigned long long fd = 0, sd = 0;
    for (int d = 0; d < D; d++) {
      const char *b = a.bufs + (size_t)d * a.L.bytes;
      int len = 0, more = 0;
      if (s < ns) {
        len = reinterpret_cast<const int *>(b + a.L.off_len)[s];
        more = reinterpret_cast<const int *>(b + a.L.off_more)[s];
        fit += reinterpret_cast<const int *>(b + a.L.off_fit)[s];
        fd += reinterpret_cast<const unsigned long long *>(b + a.L.off_fd)[s];
        sd += reinterpret_cast<const unsigned long long *>(b + a.L.off_sd)[s];
        if (len > rke) { len = rke; more = 1; }                  // the part of the list held in shared memory
      }
      S.cur[s][d] = 0; S.len[s][d] = (uint8_t)len; S.more[s][d] = (uint8_t)more; S.hkey[s][d] = 0;
    }
    S.afit[s] = fit; S.afd[s] = fd; S.asd[s] = sd; S.observed[s] = 0; S.pu[s] = -1;
    S.xbest[s] = 0; S.xbest_t[s] = -1; S.hv_nT[s] = -1; S.hpay_node[s] = -1; S.bh[s] = 0; S.bh_d[s] = 0; S.dbound[s] = 0;
    if (s < ns) {
      S.reqs[s] = a.rd->reqs[s];
      const Req &r = a.rd->reqs[s];
      S.rq_single[s] = req_is_single(r); S.rq_core[s] = r.core[0]; S.rq_mem[s] = r.mem[0];
      S.rq_cmask[s] = r.C >= 4 ? 0xFFFFFFFFu : ((1u << (8 * r.C)) - 1u);   // alloc planes >= C are never written
    }
  }
  for (int e = tid; e < ns * D * rke; e += nthreads) {
    const int k = e % rke, sd = e / rke, d = sd % D, s = sd / D;
    const int len = reinterpret_cast<const int *>(a.bufs + (size_t)d * a.L.bytes + a.L.off_len)[s];
    lk[e] = k < len ? cand_at(a.bufs, a.L, d, s, k).key() : 0ull;
  }
  __syncthreads();
  n_pre = 0;
  if constexpr (I::kPreinstall) {
    if (tid < 32) {
      const int n = preinstall_select(S, a, lk, psrc, ns, tid);
      if (tid == 0) S.nT = n;
    }
    __syncthreads();
    n_pre = S.nT;
    preinstall_slots(S, a, psrc, n_pre, ns);
    for (int i = tid; i < NS * RD; i += nthreads) (&S.cur[0][0])[i] = 0;   // the owners' list cursors start at the top
  }
  if (tid == 0) {
    // Monotone round: every container fractional with requests >= 0.  Rows then only decrease, and fractional
    // feasibility (avail >= request) is monotone in the rows.  A whole-GPU container tests EQUALITY with the totals
    // (gpu.go:193-202): a GPU above its totals (a sidecar's +1, ForgetPod after a failed AddPod, a loaded row) is
    // not free, and a bind that brings it down to its totals frees it -- so a round with one is never monotone.
    bool mono = true;
    for (int s = 0; s < ns; s++)
      for (int c = 0; c < S.reqs[s].C; c++) mono &= S.reqs[s].core[c] >= 0 && S.reqs[s].mem[c] >= 0 && S.reqs[s].cnt[c] == 0;
    S.mono = mono ? 1 : 0;
  }
  __syncthreads();
  return true;
}

template <class SM>
__device__ __noinline__ void resolve_epilogue(SM &S, const MwArgs &a) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nthreads = blockDim.x;
  const int ns = a.rd->ns;
  const int p0 = S.p0;
  // ---- epilogue: write the tracked nodes back (each shard its own nodes)
  const int nT = S.nT;
  const int done = S.stop_p - p0;
  const int nwarps = nthreads >> 5;
  for (int t = warp; t < nT; t += nwarps) {
    const int w = S.node[t];
    if (w < a.lo || w >= a.hi) continue;
    if (S.dirty[t]) {
      if (lane < EGS_G) a.core[(size_t)w * EGS_G + lane] = S.rc[t][lane];
      else if (lane < 2 * EGS_G) a.mem[(size_t)w * EGS_G + lane - EGS_G] = S.rm[t][lane - EGS_G];
    }
    for (int s = lane; s < ns; s += 32) {
      const int slot = a.rd->slot[s];
      const uint8_t st = S.st[s][t];
      tb_st(a.tb, slot)[w] = st;
      if (st == OPT_CACHED || st == OPT_NEW) {
        tb_sc(a.tb, slot)[w] = key_score(S.tkey[s][t]);
        uint8_t *alp = tb_al(a.tb, slot);
        const uint32_t am = S.al[s][t];
        for (int c = 0; c < S.reqs[s].C; c++) alp[(size_t)c * a.tb.n_pad + w] = (uint8_t)(am >> (8 * c));
      }
    }
    if (S.dirty[t]) {                                            // shapes outside the round set
      for (int slot = lane; slot < a.tb.n_slots; slot += 32) {
        bool in_set = false;
        for (int q = 0; q < ns; q++) in_set |= a.rd->slot[q] == slot;
        if (in_set) continue;
        uint8_t *q = tb_st(a.tb, slot) + w;
        if (*q == OPT_UNFIT) *q = OPT_ABSENT;
        else if (*q == OPT_NEW) *q = a.obs_pending[slot] ? OPT_CACHED : OPT_ABSENT;
      }
    }
  }
  for (int s = tid; s < ns; s += nthreads) if (S.observed[s]) a.obs_pending[a.rd->slot[s]] = 1;
  if (tid == 0) {
    RoundCtl *c = a.ctl;
    c->next_p = p0 + done;
    if (done < 1) c->error = 1;                                  // no progress: the host reports it
    c->rounds += 1; c->pods += done; c->tracked += nT;
    c->stops[S.stop ? (S.stop_reason & 3) : 0] += 1;
  }
}

template <class I>
__global__ void __launch_bounds__(32 * MW_MAX_WARPS, 1) k_resolve_mw(MwArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using SM = typename I::Smem;
  SM &S = *reinterpret_cast<SM *>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int D = a.n_shards, rke = a.rke, nw = a.nw;
  const int ns = a.rd->ns;
  const MwTail tail = mw_tail<I>(ns, D, rke, a.L.cand_bytes);
  unsigned long long *lk = reinterpret_cast<unsigned long long *>(smem_raw + tail.lk);
  char *hpay = I::kHpay ? reinterpret_cast<char *>(smem_raw + tail.hpay) : nullptr;
  int *psrc = reinterpret_cast<int *>(smem_raw + tail.psrc);
  // what the owner loop reads of `a`, in registers: `a` is passed by reference to the non-inlined helpers, so its
  // fields otherwise live in a stack copy and every use is a local-memory load on the ordered chain
  const int policy = a.policy;
  const uint8_t *const pod_sidx = a.pod_sidx;
  int n_pre;
  if (!resolve_prologue<I>(S, a, lk, psrc, n_pre)) return;
  const int p0 = S.p0, p_end = S.p_end;
#ifdef EGS_RESOLVE_PROF
  long long prof[RPROF]; for (int i = 0; i < RPROF; i++) prof[i] = 0;
  long long tprev = clock64();
#endif
  // ---- the owner loop.  Pods of shapes si with si % nw == warp, in pod order.
  if (warp < nw) {
    // own pods are found 128 at a time: lane loads 4 shape indices
    int cb = p0 & ~3;                                            // chunk base (multiple of 4)
    unsigned pm[4] = {0, 0, 0, 0};                               // per j: lanes whose pod 4*lane+j is mine
    uint32_t myword = 0;
    uint32_t nextword = 0xFFFFFFFFu, prevword = 0xFFFFFFFFu;     // shape indices of pods cb+128..cb+131 / cb-4..cb-1
    unsigned ph = 0;                                             // phase parity of my mbarrier
    auto load_chunk = [&](int base) {
      const int q = base + 4 * lane;
      uint32_t wd = 0xFFFFFFFFu;
      if (q < p_end) wd = *reinterpret_cast<const uint32_t *>(pod_sidx + q);   // padded allocation: reads up to 3 past the end
      myword = wd;
      uint32_t nx = 0xFFFFFFFFu, pv = 0xFFFFFFFFu;
      if (lane == 0 && base + 128 < p_end) nx = *reinterpret_cast<const uint32_t *>(pod_sidx + base + 128);
      if (lane == 0 && base >= 4) pv = *reinterpret_cast<const uint32_t *>(pod_sidx + base - 4);
      nextword = __shfl_sync(0xffffffffu, nx, 0); prevword = __shfl_sync(0xffffffffu, pv, 0);
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int si = (wd >> (8 * j)) & 0xFF;
        const bool mine = (q + j >= p0) && (q + j < p_end) && si < ns && (si % nw) == warp;
        pm[j] = __ballot_sync(0xffffffffu, mine);
      }
    };
    load_chunk(cb);
    // owner of pod cb + i (i in [-4, 131]); -1 outside [p0, p_end).  Warp-uniform, all lanes call it.
    auto owner_rel = [&](int i) -> int {
      const uint32_t wd = __shfl_sync(0xffffffffu, myword, (i >> 2) & 31);
      const uint32_t x = i < 0 ? prevword : i >= 128 ? nextword : wd;
      const int si = (int)((x >> (8 * (i & 3))) & 0xFFu);
      return (cb + i >= p0 && cb + i < p_end && si < ns) ? si % nw : -1;
    };
    const bool mono = S.mono != 0;
    const int gl = lane & 7;
    while (true) {
      // next own pod
      int p = -1, s = 0, wake = -1; bool sleep_first = false;
      while (true) {
        int best_i = 1 << 30;
#pragma unroll
        for (int j = 0; j < 4; j++) if (pm[j]) { const int i = 4 * (__ffs(pm[j]) - 1) + j; best_i = min(best_i, i); }
        if (best_i < (1 << 30)) {
          const int j = best_i & 3, l = best_i >> 2;
#pragma unroll
          for (int jj = 0; jj < 4; jj++) if (jj == j) pm[jj] &= ~(1u << l);   // static indices: pm stays in registers
          p = cb + best_i;
          s = (__shfl_sync(0xffffffffu, myword, l) >> (8 * j)) & 0xFF;
          // whom do I wake after my ticket (the owner of p + 1 unless that is me), and do I sleep before mine?
          wake = owner_rel(best_i + 1);                           // the next owner sleeps on its mbarrier until I arrive
          sleep_first = p > p0 && owner_rel(best_i - 1) != warp;  // exactly one arrive per wait
          if (wake == warp) wake = -1;
          break;
        }
        cb += 128;
        if (cb >= p_end) break;
        load_chunk(cb);
      }
      if (p < 0) break;
      PROF_T(22)
      // ======== preparation outside the ticket: only owner-private data and data that never changes
      maintain_heads(S, lk, D, rke, s, lane, false);
      PROF_T(23)
      const unsigned long long head = S.bh[s];
      if constexpr (I::kHpay) {
        if (head != 0 && S.hpay_node[s] != (int)key_node(head)) {         // payload of the best head -> shared memory,
          const int d = S.bh_d[s];                                        // asynchronously: only a head-win waits for it
          const char *src = cand_at(a.bufs, a.L, d, s, S.cur[s][d]).p;
          char *dst = hpay + (size_t)s * a.L.cand_bytes;
          asm volatile("cp.async.wait_all;" ::: "memory");                // an older copy into this buffer has long landed
          for (int i = lane; i < a.L.cand_bytes / 16; i += 32)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst + i * 16)), "l"(src + i * 16) : "memory");
          asm volatile("cp.async.commit_group;" ::: "memory");
          __syncwarp();                                                   // every lane has compared hpay_node
          if (lane == 0) S.hpay_node[s] = (int)key_node(head);
          __syncwarp();
        }
      }
      PROF_T(24)
      // n_observed BEFORE pu: other warps write pu[s] / the aggregates of s (general_pod, inside their tickets) only while
      // some shape of the round is unobserved; once n_observed == ns was seen, everything read below is owner-private
      const int n_obs = ld_vol(&S.n_observed);
      const int pu = ld_vol(&S.pu[s]);
      const bool fast = mono && S.rq_single[s] && pu != -2 && n_obs == ns;
      // fast pods: the best tracked option of s over the slots seen so far, and everything the ticket will need
      unsigned long long pre_best = 0; int pre_t = -1;
      const int u = pu, uu = max(pu, 0);
      uint32_t und = 0, pre_al = 0; unsigned long long ft_u = 0, sb_u = 0, afd = 0, asd = 0, dbp = 0;
      int rq_c = 0, rq_m = 0, afit = 0, v_pre = -1, bk_pre = -1;
      if (fast) {
        const int pre_nT = ld_vol(&S.nT);
        __threadfence_block();
        unsigned long long b = 0; int bt = -1;
#pragma unroll 4
        for (int t = lane; t < pre_nT; t += 32) { const unsigned long long k = S.tkey[s][t]; if (k > b) { b = k; bt = t; } }
        int owner;
        pre_best = warp_max_key_fwd(b, owner);
        pre_t = __shfl_sync(0xffffffffu, bt, owner);
        pre_al = pre_t >= 0 ? (S.al[s][pre_t] & 0xFFu) : 0u;
        und = (uint32_t)S.node[uu]; ft_u = S.fterm[uu]; sb_u = S.sbase[uu];
        rq_c = S.rq_core[s]; rq_m = S.rq_mem[s];
        afit = S.afit[s]; afd = S.afd[s]; asd = S.asd[s]; dbp = S.dbound[s];
        if (u >= 0) {                                             // Trade of the pending option on the rows as they are NOW;
          v_pre = ld_vol(&S.ver[uu]);                             // the ticket reuses it when no bind touched the node since
          int c[EGS_G], m[EGS_G];
#pragma unroll
          for (int g = 0; g < EGS_G; g++) { c[g] = ld_vol(&S.rc[uu][g]); m[g] = ld_vol(&S.rm[uu][g]); }
          bk_pre = trade_lanes(c, m, gl, rq_c, rq_m, policy);
          if ((v_pre & 1) || ld_vol(&S.ver[uu]) != v_pre) v_pre = -1;   // a bind was writing the rows meanwhile
        }
      }
      PROF_T(0)
#ifdef EGS_RESOLVE_PROF
      const bool late_ = sleep_first && ld_vol(&S.turn) == p;     // the ticket was already open: it waited for my preparation
#endif
      // ======== the ticket
      bool stopped = false;
      if (sleep_first) {                                          // else: I still hold the ticket
        while (!mbar_try_wait(&S.mbar[warp], ph)) { if (ld_vol(&S.turn) & MW_STOP) { stopped = true; break; } }
        ph ^= 1u;
        if (ld_vol(&S.turn) & MW_STOP) stopped = true;
      }
      if (stopped) break;
      PROF_T(1)
#ifdef EGS_RESOLVE_PROF
      if (p > p0) {                                               // release of pod p-1 -> start of pod p, on the chain
        const long long gap_ = tprev - *reinterpret_cast<volatile long long *>(&S.t_release);
        if (!sleep_first) { prof[18] += gap_; prof[19] += 1; }    // kept the ticket: my own post + preparation
        else if (late_) { prof[20] += gap_; prof[21] += 1; }      // handed over to an owner that was not ready
        else { prof[16] += gap_; prof[17] += 1; }                 // handed over to an owner asleep on its mbarrier
      }
#endif
      int reason = 0;
      if (fast) {
        // ---- fast pod: single-container shape, monotone round, every shape observed, at most one pending option
        const unsigned long long xb = S.xbest[s];
        const int xt = S.xbest_t[s];
        int bk = bk_pre;
        if (u >= 0 && S.ver[uu] != v_pre) {                       // the node's rows changed since the preparation
          const int4 c0 = *reinterpret_cast<const int4 *>(&S.rc[uu][0]), c1 = *reinterpret_cast<const int4 *>(&S.rc[uu][4]);
          const int4 m0 = *reinterpret_cast<const int4 *>(&S.rm[uu][0]), m1 = *reinterpret_cast<const int4 *>(&S.rm[uu][4]);
          const int c[EGS_G] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
          const int m[EGS_G] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
          bk = trade_lanes(c, m, gl, rq_c, rq_m, policy);
          PROF_C(14, 1)
        }
#ifdef EGS_RESOLVE_PROF
        long long q1_ = clock64() + (bk & 0);
#endif
        const int sc = (bk >= 0 && policy == EGS_BINPACK) ? (bk >> 3) * 100 : 0;
        const unsigned long long tradekey = bk >= 0 ? cand_key(sc, und) : 0ull;
        unsigned long long best = pre_best; int tw = pre_t; uint32_t masks = pre_al;
        if (xb > best) { best = xb; tw = xt; masks = 0; }
        if (tradekey > best) { best = tradekey; tw = u; masks = 1u << (bk & 7); }
        // Exact rule (head*, dbound* = the exact values at this ticket): dbound* > max(head*, best) -> the round ends;
        // head* > best -> head-win; else a tracked option wins.  head / dbp were taken during the preparation; both only
        // shrink over time and a list exhausted since then ends below the head it had then, so:
        //   best >= max(head, dbp)                      -> tracked win (nothing untracked can beat it)
        //   head <= best < dbp                          -> dbound* >= dbp > best >= head*: the round ends
        //   head > best, head's node still untracked    -> head* == head; dbound* > head* iff dbp > head
        //   head > best, head's node tracked by now     -> re-validate the lists inside the ticket (exact) and apply the rule
        // -- the same outcome whatever the timing of the preparation: replicated resolvers stay in lock step.
        unsigned long long hd = head;
        if ((hd > dbp ? hd : dbp) > best) {
          if (hd <= best) reason = 3;
          else if (!hset_has(S, key_node(hd))) { if (dbp > hd) reason = 3; }
          else {
            maintain_heads(S, lk, D, rke, s, lane, true);
            hd = S.bh[s];
            if (S.dbound[s] > (hd > best ? hd : best)) reason = 3;
            PROF_C(15, 1)
          }
        }
        const bool from_head = reason == 0 && hd > best;
        const unsigned long long win = from_head ? hd : best;
        int nT = 0;
        if (from_head) { nT = S.nT; if (nT >= I::NT) reason = 2; }
#ifdef EGS_RESOLVE_PROF
        long long q2_ = clock64() + (reason & 0) + ((int)win & 0);
        long long q3_ = q2_;
#endif
        if (reason == 0) {
          int o_node = -1, o_status = EGS_ERR_NOFIT; uint32_t o_masks = 0;
          if (win != 0) {
            if (from_head) {
              tw = nT;
              const uint32_t w = key_node(win);
              asm volatile("cp.async.wait_all;" ::: "memory");
              __syncwarp();
              install_slot(S, head_payload(S, a, hpay, s, w), tw, w, ns, s, lane);
              __syncwarp();
              masks = S.al[s][tw] & 0xFFu;
              PROF_C(11, 1)
            } else if (masks == 0) {
              masks = S.al[s][tw] & 0xFFu;                        // a slot another shape installed
            }
            o_node = S.node[tw];
            const int ok = bind_single_slot(S, tw, __ffs(masks) - 1, rq_c, rq_m, lane);
#ifdef EGS_RESOLVE_PROF
            q3_ = clock64() + (ok & 0) + (o_node & 0);
#endif
            o_status = ok ? EGS_OK : EGS_ERR_TRANSACT; o_masks = ok ? masks : 0;
          }
          // ---- hand the ticket on (arrive = release), then the owner-private part
          if (lane == 0) {
            if (from_head) { __threadfence_block(); st_vol(&S.nT, nT + 1); }
            if (xb != 0) { S.xbest[s] = 0; S.xbest_t[s] = -1; }
            st_vol(&S.turn, p + 1);
            PROF_RELEASE()
            if (wake >= 0) mbar_arrive(&S.mbar[wake]);
          }
#ifdef EGS_RESOLVE_PROF
          { const long long n_ = clock64(); prof[from_head && win != 0 ? 5 : 2] += n_ - tprev;
            if (!(from_head && win != 0)) { prof[7] += q1_ - tprev; prof[8] += q2_ - q1_; prof[10] += q3_ - q2_; prof[12] += n_ - q3_; }
            tprev = n_; }
#endif
          PROF_C(6, 1)
          const int fit = afit + (bk >= 0);
          const unsigned long long fd = afd + (bk >= 0 ? ft_u : 0ull);
          const unsigned long long sd = asd + (bk >= 0 ? score_term_b(sb_u, sc) : 0ull);
          if (lane == 0) {
            if (u >= 0 && u != tw) {                              // this pod's filter Traded slot u
              if (bk >= 0) { S.st[s][u] = OPT_CACHED; S.al[s][u] = 1u << (bk & 7); S.tkey[s][u] = tradekey; }
              else S.st[s][u] = OPT_UNFIT;
              S.pmask[s][u >> 5] &= ~(1u << (u & 31));
            }
            if (win != 0) consume_option(S, s, tw, win, fit, fd, sd);
            else { S.afit[s] = fit; S.afd[s] = fd; S.asd[s] = sd; S.pu[s] = -1; }
            write_pod_out<EGS_G>(a.out, p, o_node, o_status, fit, fd, sd, o_masks);
          }
          __syncwarp();
          PROF_T(3)
          continue;
        }
      } else {
        reason = general_pod(S, a, lk, hpay, lane, p, s, ns);
        PROF_C(9, 1)
      }
      if (reason) {                                               // the round ends BEFORE pod p: wake every owner
        if (lane == 0) { S.stop_reason = reason; S.stop_p = p; S.stop = 1; st_vol(&S.turn, p | MW_STOP); }
        __syncwarp();
        if (lane < nw && lane != warp) mbar_arrive(&S.mbar[lane]);
        break;
      }
      __syncwarp();
      if (lane == 0) { st_vol(&S.turn, p + 1); PROF_RELEASE() if (wake >= 0) mbar_arrive(&S.mbar[wake]); }
      PROF_T(4)
    }
  }
  __syncthreads();
  resolve_epilogue(S, a);
#ifdef EGS_RESOLVE_PROF
  if (warp == 0) prof[13] += n_pre;                             // pre-installed slots
  if (lane == 0 && warp < nw) for (int i = 0; i < RPROF; i++) atomicAdd((unsigned long long *)&a.ctl->prof[i], (unsigned long long)prof[i]);
#endif
}

// End of a ROUNDS batch: no OPT_NEW may outlive it (the other code paths know three states).
__global__ void k_rounds_finalize(TableSet tb, uint8_t *obs_pending, int lo, int hi) {
  const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= hi) return;
  for (int slot = 0; slot < tb.n_slots; slot++) {
    uint8_t *q = tb_st(tb, slot) + i;
    if (*q == OPT_NEW) *q = obs_pending[slot] ? OPT_CACHED : OPT_ABSENT;
  }
}
__global__ void k_clear_u8(uint8_t *p, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0;
}

// ---------------------------------------------------------------------------------------------
struct egs_handle;

// In-process shard group (several handles, one per shard, in ONE process; typically all on one device): the
// per-round exchange is a device-to-device copy of every peer's candidate buffer ordered by CUDA events, with a host
// barrier between the threads that drive the handles.  Same data path as the NCCL exchange; lets a single-GPU box
// run (and test) the sharded engine at world sizes 2..8.
struct LocalGroup {
  int world = 0;
  std::vector<egs_handle *> members;
  std::mutex mu; std::condition_variable cv; int arrived = 0; long long generation = 0;
  bool broken = false;
  bool barrier() {                                   // false: a member never came (its batch failed): the group is broken
    std::unique_lock<std::mutex> lk(mu);
    if (broken) return false;
    const long long g = generation;
    if (++arrived == world) { arrived = 0; generation++; cv.notify_all(); return true; }
    if (!cv.wait_for(lk, std::chrono::seconds(60), [&] { return generation != g || broken; })) { broken = true; cv.notify_all(); }
    return !broken;
  }
};

struct RoundsState {
  void *comm = nullptr;             // ncclComm_t
  std::shared_ptr<LocalGroup> local;                    // in-process shard group (instead of NCCL)
  cudaEvent_t ev_ready = nullptr, ev_copied = nullptr;   // own buffer written / peers' buffers copied
  bool copied = false;              // in-process group: a round ran since egs_comm_init_local, so every peer's
                                    // ev_copied marks its last copy of this rank's buffer (kept across batches)
  DeviceBuf<uint8_t> d_pod_sidx;
  DeviceBuf<uint8_t> d_obs;
  DeviceBuf<unsigned long long> d_cta_lists; DeviceBuf<AggPart> d_cta_agg; int grid = 0, cta_nsc = 0;
  DeviceBuf<char> d_bufs;                           // [RD] candidate buffers; own shard written at index `rank`
  DeviceBuf<RoundDesc> d_rd; PinnedBuf<RoundDesc> h_rd;
  DeviceBuf<RoundCtl> d_ctl; PinnedBuf<RoundCtl> h_ctl;
  int64_t rounds = 0, pods = 0, tracked = 0; int64_t stops[4] = {0, 0, 0, 0};
  long long prof[RPROF] = {0};
};

static int batch_rescan(egs_handle *h, int P, const int32_t *c_off, const egs_unit *units,
                        const std::vector<int> &slots, PodOut out, const uint64_t *d_set);
static int batch_rounds(egs_handle *h, int P, const std::vector<int> &slots, PodOut out, int *n_done,
                        const uint64_t *d_set);
static void rounds_free(RoundsState *r);
static int rounds_comm_unique_id(uint8_t out_id[128]);
static int rounds_comm_init(egs_handle *h, const uint8_t id[128]);
static int rounds_comm_init_local(egs_handle **handles, int world);
