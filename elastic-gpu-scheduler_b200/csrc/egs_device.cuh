// egs_device.cuh -- device-side GPU/GPUs arithmetic of the reference's L0 layer
// (pkg/scheduler/{gpu,rater}.go) on the int32 SoA rows.  Pure integer work.
//
// A node's row is free_core[G], free_mem[G] with G = EGS_ROW_WIDTH(g_max) (8, or 16 on a wide handle); GPUs a node
// does not have hold
// EGS_PAD in BOTH arrays.  EGS_PAD = INT32_MIN fails every CanAllocate test
// (requests are >= -1, gpu.go:51-56) and is skipped by the Rate min/max scan,
// so no per-node gpu_count has to be read on the hot path.
#pragma once
#include <stdint.h>
#include "../../include/egs.h"

// The arithmetic below is also compiled for the HOST (tests/test_device_arith_host.py runs it against
// the oracle without a GPU); device intrinsics are spelled through these macros.
#ifdef __CUDA_ARCH__
#define EGS_HD __host__ __device__ __forceinline__
#define EGS_MAX3(a, b, c) __vimax3_s32((a), (b), (c))
#define EGS_POPC(x) __popc(x)
#define EGS_FFS(x) __ffs(x)
#define EGS_MIN(a, b) min((a), (b))
#define EGS_MAX(a, b) max((a), (b))
#else
#include <algorithm>
#define EGS_HD __host__ __device__ inline
#define EGS_MAX3(a, b, c) std::max(std::max((a), (b)), (c))
#define EGS_POPC(x) __builtin_popcount(x)
#define EGS_FFS(x) __builtin_ffs((int)(x))
#define EGS_MIN(a, b) std::min((a), (b))
#define EGS_MAX(a, b) std::max((a), (b))
#endif

#define EGS_PAD INT32_MIN
#define EGS_G EGS_MAX_GPUS
#define EGS_C EGS_MAX_CONTAINERS

// option-cache entry states (node.go:19 `allocated map[string]*GPUOption`)
#define OPT_ABSENT 0  // no entry: the next filter Trades this node
#define OPT_CACHED 1  // entry present: reused verbatim, even if stale (node.go:64-66)
#define OPT_UNFIT  2  // memo: Trade failed on the CURRENT rows (cleared whenever the rows change);
                      // the reference re-Trades such nodes every time with the same outcome

// GPURequest (allocate.go:20) for one pod, by value in kernel params / shared memory.
struct Req {
  static constexpr int NC = EGS_C;   // containers the type holds: the option masks of a pod are NC planes
  int C;
  int core[EGS_C];
  int mem[EGS_C];
  int cnt[EGS_C];
};
#define EGS_CA EGS_MAX_CONTAINERS_APPLY
// a pod as AddPod / ForgetPod see it, and as a sidecar handle (c_max > 4) Trades it: up to 8 containers
struct ReqW { static constexpr int NC = EGS_CA; int C; int core[EGS_CA], mem[EGS_CA], cnt[EGS_CA]; };

// Req or ReqW from C units (C within the type's bound, checked by the caller); unused containers are zero.
template <class R = Req>
inline R make_req(int C, const egs_unit *u) {
  R r = {};
  r.C = C;
  for (int i = 0; i < C; i++) { r.core[i] = u[i].core; r.mem[i] = u[i].mem; r.cnt[i] = u[i].count; }
  return r;
}

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  uint64_t z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ uint64_t fit_term(uint32_t node) { return mix64(2ull * node + 1ull); }
// score digest term = h2(node) * (2*score + 1): h2 is per node, so it is hashed once and reused for every shape
__host__ __device__ __forceinline__ uint64_t score_base(uint32_t node) { return mix64(2ull * node + 2ull); }
__host__ __device__ __forceinline__ uint64_t score_term_b(uint64_t base, int32_t score) {
  return base * (2ull * (uint64_t)(uint32_t)score + 1ull);
}
__host__ __device__ __forceinline__ uint64_t score_term(uint32_t node, int32_t score) {
  return score_term_b(score_base(node), score);
}
// candidate ordering: higher score first, then lower node id ("first max in list order").
// Scores are >= 0 (rater.go:49-50 with operands >= 0), so key 0 means "no candidate".
__host__ __device__ __forceinline__ uint64_t cand_key(int32_t score, uint32_t node) {
  return ((uint64_t)(uint32_t)score << 32) | (uint64_t)(0xFFFFFFFFu - node);
}
__host__ __device__ __forceinline__ uint32_t key_node(uint64_t key) { return 0xFFFFFFFFu - (uint32_t)key; }
__host__ __device__ __forceinline__ int32_t key_score(uint64_t key) { return (int32_t)(key >> 32); }

// Per row width G: the GPU mask of one container (Mask), and LG = log2(G) for the folded Trade keys.
template <int G> struct RowWidth;
template <> struct RowWidth<8> { typedef uint8_t Mask; static constexpr int LG = 3; };
template <> struct RowWidth<16> { typedef uint16_t Mask; static constexpr int LG = 4; };
template <int G> using MaskT = typename RowWidth<G>::Mask;
// Per geometry (row width G, NP mask planes per pod): the masks of a pod's NP containers packed into one word
// (container k at bits [G*k, G*k + G)).  Three geometries exist: (8, 4) and (16, 4), and (8, 8) on a sidecar handle.
template <int G, int NP> struct Geometry;
template <> struct Geometry<8, EGS_C> { typedef uint32_t Packed; typedef Req R; };
template <> struct Geometry<16, EGS_C> { typedef uint64_t Packed; typedef Req R; };
template <> struct Geometry<8, EGS_CA> { typedef uint64_t Packed; typedef ReqW R; };
template <int G, int NP = EGS_C> using PackedT = typename Geometry<G, NP>::Packed;
template <int NP> using ReqOf = typename Geometry<EGS_G, NP>::R;

// G/4 16-byte read-only loads per array: one node's row (4*G B core + 4*G B mem), all issued before any use.
template <int G>
__device__ __forceinline__ void load_row(const int32_t *__restrict__ core, const int32_t *__restrict__ mem,
                                         size_t node, int (&c)[G], int (&m)[G]) {
  const int4 *pc = reinterpret_cast<const int4 *>(core + node * G);
  const int4 *pm = reinterpret_cast<const int4 *>(mem + node * G);
  int4 cv[G / 4], mv[G / 4];
#pragma unroll
  for (int q = 0; q < G / 4; q++) cv[q] = __ldg(pc + q);
#pragma unroll
  for (int q = 0; q < G / 4; q++) mv[q] = __ldg(pm + q);
#pragma unroll
  for (int q = 0; q < G / 4; q++) {
    c[4 * q] = cv[q].x; c[4 * q + 1] = cv[q].y; c[4 * q + 2] = cv[q].z; c[4 * q + 3] = cv[q].w;
    m[4 * q] = mv[q].x; m[4 * q + 1] = mv[q].y; m[4 * q + 2] = mv[q].z; m[4 * q + 3] = mv[q].w;
  }
}

// ---------------------------------------------------------------------------------------------
// Fast Trade: one container, fractional unit with core >= 0 and mem >= 0 (GPUCount == 0).
// gpu.go:110-122 tries GPU 0..G-1; the leaf keeps the option unless best > score (gpu.go:85),
// so the LAST maximal GPU wins.  Binpack.Rate (rater.go:18-51) needs min/max over all rows
// after the Add on GPU g:
//   * new value n = row[g] - req <= row[g], so  min' = min(min_all, n)           (no exclusion needed)
//   * max' = max(max over rows != g, n): prefix/suffix maxima + one 3-input max
//   * PAD (INT32_MIN) is the smallest signed value: a signed max ignores absent GPUs without a select, the min
//     skips them.  Rows can be negative -- ForgetPod of a sentinel unit takes 1 from a GPU (gpu.go:41-49) -- so the
//     min is a signed one, as Go's.
//   * score = Range/(1+1)*100 with Range = x/2, x >= 0  ==  (x >> 2) * 100        (rater.go:49-50)
//   * candidates are folded as key = q*G + g: one max keeps the last maximal GPU.  q = x >> 2 with
//     x <= 2*(EGS_MAX_MEM_PER_GPU + EGS_MAX_CORE_LOAD) < 2^26.1, so q < 2^24.1 and the largest key,
//     q*16 + 15, stays below 2^28: no int32 overflow at G = 16 under the load / unit guards.
// Returns true when some GPU fits; score / gpu index by reference.
// ---------------------------------------------------------------------------------------------
template <int G>
EGS_HD bool trade_single(const int (&c)[G], const int (&m)[G], int rc, int rm,
                         int policy, int &score, int &gidx) {
  constexpr int LG = RowWidth<G>::LG;
  int bestkey = -1;
  if (policy == EGS_BINPACK) {
    int cmin = INT32_MAX, mmin = INT32_MAX;
    int cpre[G], csuf[G], mpre[G], msuf[G];
    cpre[0] = INT32_MIN; mpre[0] = INT32_MIN; csuf[G - 1] = INT32_MIN; msuf[G - 1] = INT32_MIN;
#pragma unroll
    for (int g = 0; g < G; g++) {
      const bool real = c[g] != EGS_PAD;
      cmin = real ? EGS_MIN(cmin, c[g]) : cmin; mmin = real ? EGS_MIN(mmin, m[g]) : mmin;
    }
#pragma unroll
    for (int g = 1; g < G; g++) { cpre[g] = EGS_MAX(cpre[g - 1], c[g - 1]); mpre[g] = EGS_MAX(mpre[g - 1], m[g - 1]); }
#pragma unroll
    for (int g = G - 2; g >= 0; g--) { csuf[g] = EGS_MAX(csuf[g + 1], c[g + 1]); msuf[g] = EGS_MAX(msuf[g + 1], m[g + 1]); }
#pragma unroll
    for (int g = 0; g < G; g++) {
      const bool ok = (c[g] >= rc) && (m[g] >= rm);         // CanAllocate gpu.go:55; PAD rows fail
      const int nc = c[g] - rc, nm = m[g] - rm;             // GPU.Add gpu.go:36-37
      const int cmx = EGS_MAX3(cpre[g], csuf[g], nc), cmn = EGS_MIN(cmin, nc);
      const int mmx = EGS_MAX3(mpre[g], msuf[g], nm), mmn = EGS_MIN(mmin, nm);
      const int x = (mmx + cmx) - (mmn + cmn);
      const int key = ok ? ((x >> 2) * G + g) : -1;
      bestkey = EGS_MAX(bestkey, key);
    }
    score = (bestkey >> LG) * 100;
  } else {                                                   // Spread.Rate == 0 (rater.go:56-59): last feasible GPU
#pragma unroll
    for (int g = 0; g < G; g++) bestkey = ((c[g] >= rc) && (m[g] >= rm)) ? g : bestkey;
    score = 0;
  }
  gidx = bestkey & (G - 1);
  return bestkey >= 0;
}

// The same Trade as trade_single, one GPU per lane (the resolver's form: the lane holds the whole row, gl = its GPU).
// Returns the lane's folded key -- (x >> 2) * 8 + gl under binpack, gl under spread, -1 when GPU gl does not fit;
// the max over gl = 0..7 is trade_single's bestkey.  The max over the OTHER GPUs is a masked scan of the row.
EGS_HD int trade_lane_key(const int (&c)[EGS_G], const int (&m)[EGS_G], int gl, int rq_c, int rq_m, int policy) {
  int cmin = INT32_MAX, mmin = INT32_MAX;
  int cex = INT32_MIN, mex = INT32_MIN, cg = 0, mg = 0;
#pragma unroll
  for (int g = 0; g < EGS_G; g++) {
    const bool real = c[g] != EGS_PAD;                           // signed min over the GPUs present (trade_single)
    cmin = real ? EGS_MIN(cmin, c[g]) : cmin; mmin = real ? EGS_MIN(mmin, m[g]) : mmin;
    cex = EGS_MAX(cex, g == gl ? INT32_MIN : c[g]); mex = EGS_MAX(mex, g == gl ? INT32_MIN : m[g]);
    cg = g == gl ? c[g] : cg; mg = g == gl ? m[g] : mg;
  }
  const bool ok = cg >= rq_c && mg >= rq_m;                      // CanAllocate gpu.go:55; PAD rows fail
  const int nc = cg - rq_c, nm = mg - rq_m;                      // GPU.Add gpu.go:36-37
  const int x = (EGS_MAX(mex, nm) + EGS_MAX(cex, nc)) - (EGS_MIN(mmin, nm) + EGS_MIN(cmin, nc));
  return !ok ? -1 : (policy == EGS_BINPACK ? (x >> 2) * 8 + gl : gl);
}

// ---------------------------------------------------------------------------------------------
// General Trade: up to R::NC containers (4, or 8 on a sidecar handle), whole-GPU units, sentinel units.  Depth-first
// over the containers exactly as gpu.go:72-123.  Cold path: rows live in local memory.
// ---------------------------------------------------------------------------------------------
template <int G, class R>
struct TradeCtx {
  typedef PackedT<G, R::NC> P;
  int c[G], m[G];
  int mem_total, policy;
  const R *r;
  P masks;              // R::NC x Mask: GPUs chosen per container on the current DFS path
  int best;
  P best_masks;
  bool found;
};

#ifdef __CUDA_ARCH__
#define EGS_HD_NOINLINE __host__ __device__ __noinline__
#else
#define EGS_HD_NOINLINE __host__ __device__ inline
#endif
template <int G, class R>
EGS_HD_NOINLINE void trade_leaf(TradeCtx<G, R> &t) {  // gpu.go:73-93
  int s = 0;
  if (t.policy == EGS_BINPACK) {
    // rateIndexes: containers holding exactly one GPU (gpu.go:76-83); k = distinct GPUs (rater.go:19-30)
    uint32_t used = 0;
#pragma unroll 1
    for (int i = 0; i < t.r->C; i++) {
      uint32_t mk = (uint32_t)(t.masks >> (G * i)) & ((1u << G) - 1u);
      if (EGS_POPC(mk) == 1) used |= mk;
    }
    int k = EGS_POPC(used);
    int cmin = INT32_MAX, cmax = INT32_MIN, mmin = INT32_MAX, mmax = INT32_MIN;
#pragma unroll 1
    for (int g = 0; g < G; g++) {
      if (t.c[g] == EGS_PAD) continue;
      cmin = EGS_MIN(cmin, t.c[g]); cmax = EGS_MAX(cmax, t.c[g]);
      mmin = EGS_MIN(mmin, t.m[g]); mmax = EGS_MAX(mmax, t.m[g]);
    }
    int range = (mmax + cmax - mmin - cmin) / 2;
    s = range / (k + 1) * 100;
  }
  t.found = true;
  if (t.best > s) return;  // gpu.go:85
  t.best = s;
  t.best_masks = t.masks;
}

template <int G, class R, int CI>
EGS_HD_NOINLINE void trade_dfs(TradeCtx<G, R> &t) {
  typedef PackedT<G, R::NC> P;
  if constexpr (CI == R::NC) {
    trade_leaf(t);
  } else {
    if (CI == t.r->C) { trade_leaf(t); return; }
    const int rc = t.r->core[CI], rm = t.r->mem[CI], cnt = t.r->cnt[CI];
    const P keep = t.masks & ~((P)MaskT<G>(~0u) << (G * CI));
    if (cnt > 0) {  // gpu.go:95-109 with GetFreeGPUs gpu.go:193-202 on the mutated rows
      uint32_t fm = 0; int nf = 0;
#pragma unroll 1
      for (int g = 0; g < G; g++)
        if (nf < cnt && t.c[g] == EGS_CORE_PER_GPU && t.m[g] == t.mem_total) { fm |= 1u << g; nf++; }
      if (nf < cnt) return;
#pragma unroll 1
      for (int g = 0; g < G; g++) if ((fm >> g) & 1u) { t.c[g] = 0; t.m[g] = 0; }          // Add gpu.go:32-34
      t.masks = keep | ((P)fm << (G * CI));
      trade_dfs<G, R, CI + 1>(t);
#pragma unroll 1
      for (int g = 0; g < G; g++) if ((fm >> g) & 1u) { t.c[g] = EGS_CORE_PER_GPU; t.m[g] = t.mem_total; }  // Sub gpu.go:42-44
      t.masks = keep;
      return;
    }
#pragma unroll 1
    for (int g = 0; g < G; g++) {  // gpu.go:110-122
      if (!(t.c[g] >= rc && t.m[g] >= rm)) continue;
      t.c[g] -= rc; t.m[g] -= rm;
      t.masks = keep | (((P)1u << g) << (G * CI));
      trade_dfs<G, R, CI + 1>(t);
      t.c[g] += rc; t.m[g] += rm;
    }
    t.masks = keep;
  }
}

template <int G, class R>
EGS_HD bool trade_general(const int (&c)[G], const int (&m)[G], int mem_total,
                          const R &r, int policy, int &score, PackedT<G, R::NC> &masks) {
  TradeCtx<G, R> t;
#pragma unroll
  for (int g = 0; g < G; g++) { t.c[g] = c[g]; t.m[g] = m[g]; }
  t.mem_total = mem_total; t.policy = policy; t.r = &r; t.masks = 0; t.best = 0; t.best_masks = 0; t.found = false;
  trade_dfs<G, R, 0>(t);
  score = t.best; masks = t.best_masks;
  return t.found;
}

// ---------------------------------------------------------------------------------------------
// Leaf-parallel form of the general Trade (the resolver evaluates the leaves of one node across the lanes of a
// warp).  The DFS of gpu.go:72-123 branches only at containers with GPUCount == 0 (one GPU each, tried in index
// order); whole-GPU containers take the first `cnt` free GPUs of the rows as mutated so far, without branching
// (gpu.go:95-109).  A leaf is therefore the tuple of GPU digits of the branching containers; DFS order ==
// lexicographic order with the FIRST branching container most significant, and "the last maximal leaf wins"
// (gpu.go:85) == the maximal (score, leaf index).  Digits are `bits` wide; a digit that names a GPU the node does
// not have meets a PAD row and fails CanAllocate like any other infeasible choice.
// Returns the leaf's score (>= 0) and its Allocated masks, or -1 when the leaf is infeasible.  The template takes
// ReqW and 64-bit masks (up to 8 containers, the leaf-split Trade of a sidecar handle); the overload after it is the
// same evaluation on Req and 32-bit masks (the resolver), kept as a plain function because the resolver kernels
// compile to a different register assignment when it is a template instance.
// With `fail`, an infeasible leaf also reports how many of its leading digits already make it infeasible: every leaf
// that shares those digits is infeasible too (trade_leaf_next skips them).  0 means no leaf of the node is feasible.
// ---------------------------------------------------------------------------------------------
template <class R, class P>
EGS_HD int trade_leaf_eval(const int (&c0)[EGS_G], const int (&m0)[EGS_G], int mem_total, const R &r, int policy,
                           int bits, int nbranch, int leaf, P &masks_out, int *fail = nullptr) {
  int c[EGS_G], m[EGS_G];
#pragma unroll
  for (int g = 0; g < EGS_G; g++) { c[g] = c0[g]; m[g] = m0[g]; }
  P masks = 0;
  uint32_t used = 0;
  int j = 0;                                                  // index among the branching containers
  for (int i = 0; i < r.C; i++) {
    if (r.cnt[i] > 0) {                                       // gpu.go:95-109 with GetFreeGPUs gpu.go:193-202
      uint32_t fm = 0; int nf = 0;
#pragma unroll
      for (int g = 0; g < EGS_G; g++) {
        const bool fr = nf < r.cnt[i] && c[g] == EGS_CORE_PER_GPU && m[g] == mem_total;
        fm |= fr ? (1u << g) : 0u; nf += fr ? 1 : 0;
      }
      if (nf < r.cnt[i]) { if (fail) *fail = j; return -1; }  // decided by the digits taken so far
#pragma unroll
      for (int g = 0; g < EGS_G; g++) { const bool t = (fm >> g) & 1u; c[g] = t ? 0 : c[g]; m[g] = t ? 0 : m[g]; }   // Add gpu.go:32-34
      masks |= (P)fm << (8 * i);
      if (EGS_POPC(fm) == 1) used |= fm;
    } else {                                                  // gpu.go:110-122
      const int gi = (leaf >> (bits * (nbranch - 1 - j))) & ((1 << bits) - 1);
      j++;
      int cg = EGS_PAD, mg = EGS_PAD;
#pragma unroll
      for (int g = 0; g < EGS_G; g++) { cg = g == gi ? c[g] : cg; mg = g == gi ? m[g] : mg; }
      if (!(cg >= r.core[i] && mg >= r.mem[i])) { if (fail) *fail = j; return -1; }   // CanAllocate gpu.go:55 (PAD rows fail)
#pragma unroll
      for (int g = 0; g < EGS_G; g++) { c[g] -= g == gi ? r.core[i] : 0; m[g] -= g == gi ? r.mem[i] : 0; }
      masks |= (P)(1u << gi) << (8 * i);
      used |= 1u << gi;
    }
  }
  masks_out = masks;
  if (policy != EGS_BINPACK) return 0;                        // Spread.Rate rater.go:56-59
  const int k = EGS_POPC(used);                               // rater.go:19-30
  int cmin = INT32_MAX, cmax = INT32_MIN, mmin = INT32_MAX, mmax = INT32_MIN;
#pragma unroll
  for (int g = 0; g < EGS_G; g++) {
    const bool real = c0[g] != EGS_PAD;
    cmin = real ? EGS_MIN(cmin, c[g]) : cmin; cmax = real ? EGS_MAX(cmax, c[g]) : cmax;
    mmin = real ? EGS_MIN(mmin, m[g]) : mmin; mmax = real ? EGS_MAX(mmax, m[g]) : mmax;
  }
  const int range = (mmax + cmax - mmin - cmin) / 2;
  return range / (k + 1) * 100;
}
EGS_HD int trade_leaf_eval(const int (&c0)[EGS_G], const int (&m0)[EGS_G], int mem_total, const Req &r, int policy,
                           int bits, int nbranch, int leaf, uint32_t &masks_out) {
  int c[EGS_G], m[EGS_G];
#pragma unroll
  for (int g = 0; g < EGS_G; g++) { c[g] = c0[g]; m[g] = m0[g]; }
  uint32_t masks = 0, used = 0;
  int j = 0;                                                  // index among the branching containers
  for (int i = 0; i < r.C; i++) {
    if (r.cnt[i] > 0) {                                       // gpu.go:95-109 with GetFreeGPUs gpu.go:193-202
      uint32_t fm = 0; int nf = 0;
#pragma unroll
      for (int g = 0; g < EGS_G; g++) {
        const bool fr = nf < r.cnt[i] && c[g] == EGS_CORE_PER_GPU && m[g] == mem_total;
        fm |= fr ? (1u << g) : 0u; nf += fr ? 1 : 0;
      }
      if (nf < r.cnt[i]) return -1;
#pragma unroll
      for (int g = 0; g < EGS_G; g++) { const bool t = (fm >> g) & 1u; c[g] = t ? 0 : c[g]; m[g] = t ? 0 : m[g]; }   // Add gpu.go:32-34
      masks |= fm << (8 * i);
      if (EGS_POPC(fm) == 1) used |= fm;
    } else {                                                  // gpu.go:110-122
      const int gi = (leaf >> (bits * (nbranch - 1 - j))) & ((1 << bits) - 1);
      j++;
      int cg = EGS_PAD, mg = EGS_PAD;
#pragma unroll
      for (int g = 0; g < EGS_G; g++) { cg = g == gi ? c[g] : cg; mg = g == gi ? m[g] : mg; }
      if (!(cg >= r.core[i] && mg >= r.mem[i])) return -1;   // CanAllocate gpu.go:55 (PAD rows fail)
#pragma unroll
      for (int g = 0; g < EGS_G; g++) { c[g] -= g == gi ? r.core[i] : 0; m[g] -= g == gi ? r.mem[i] : 0; }
      masks |= (1u << gi) << (8 * i);
      used |= 1u << gi;
    }
  }
  masks_out = masks;
  if (policy != EGS_BINPACK) return 0;                        // Spread.Rate rater.go:56-59
  const int k = EGS_POPC(used);                               // rater.go:19-30
  int cmin = INT32_MAX, cmax = INT32_MIN, mmin = INT32_MAX, mmax = INT32_MIN;
#pragma unroll
  for (int g = 0; g < EGS_G; g++) {
    const bool real = c0[g] != EGS_PAD;
    cmin = real ? EGS_MIN(cmin, c[g]) : cmin; cmax = real ? EGS_MAX(cmax, c[g]) : cmax;
    mmin = real ? EGS_MIN(mmin, m[g]) : mmin; mmax = real ? EGS_MAX(mmax, m[g]) : mmax;
  }
  const int range = (mmax + cmax - mmin - cmin) / 2;
  return range / (k + 1) * 100;
}
// The first leaf after `leaf` that does not share its first `fail` digits (trade_leaf_eval's report): nleaf when
// fail == 0.
EGS_HD int trade_leaf_next(int leaf, int fail, int bits, int nbranch) {
  const int sh = bits * (nbranch - fail);
  return ((leaf >> sh) + 1) << sh;
}
// geometry of the leaf space of request r on a node with the given rows
template <class R>
EGS_HD void trade_leaf_space(const int (&c0)[EGS_G], const R &r, int &bits, int &nbranch, int &nleaf) {
  int gcount = 0;
#pragma unroll
  for (int g = 0; g < EGS_G; g++) gcount += c0[g] != EGS_PAD ? 1 : 0;
  bits = gcount <= 1 ? 0 : gcount <= 2 ? 1 : gcount <= 4 ? 2 : 3;
  nbranch = 0;
  for (int i = 0; i < r.C; i++) nbranch += r.cnt[i] > 0 ? 0 : 1;
  nleaf = 1 << (bits * nbranch);
}

// One container, fractional, non-negative: the shape every BASELINE config except config 3 uses.
__host__ __device__ __forceinline__ bool req_is_single(const Req &r) {
  return r.C == 1 && r.cnt[0] == 0 && r.core[0] >= 0 && r.mem[0] >= 0;
}

// Trade dispatch.  `masks` packs one G-bit GPU mask per container.
template <int G, class R>
EGS_HD bool trade_any(const int (&c)[G], const int (&m)[G], int mem_total,
                      const R &r, bool single, int policy, int &score, PackedT<G, R::NC> &masks) {
  if (single) {
    int g;
    bool ok = trade_single(c, m, r.core[0], r.mem[0], policy, score, g);
    masks = (PackedT<G, R::NC>)1u << g;
    return ok;
  }
  return trade_general(c, m, mem_total, r, policy, score, masks);
}

// GPUs.Transact gpu.go:153-175 on the node's rows in global memory (one thread).
// Returns true on success; on failure the Adds already made stay (no rollback).
template <int G, class R>
EGS_HD bool transact_row(int32_t *core, int32_t *mem, int mem_total, const R &r,
                         PackedT<G, R::NC> masks) {
  for (int i = 0; i < r.C; i++) {
    uint32_t mk = (uint32_t)(masks >> (G * i)) & ((1u << G) - 1u);
    if (r.cnt[i] > 0) {
      for (int g = 0; g < G; g++) {
        if (!((mk >> g) & 1u)) continue;
        if (!(core[g] == EGS_CORE_PER_GPU && mem[g] == mem_total)) return false;
        core[g] = 0; mem[g] = 0;
      }
    } else if (mk) {
      int g = EGS_FFS(mk) - 1;
      if (!(core[g] >= r.core[i] && mem[g] >= r.mem[i])) return false;
      core[g] -= r.core[i]; mem[g] -= r.mem[i];
    }
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// Headroom of one node for one shape (egs_headroom): the binds a dry run of identical pods makes on the node.  Under
// a stream of pods of one shape a node's Assume (node.go:61-73) and Allocate (node.go:87-104) read and write only
// that node's rows and option entry, so its binds are these, in this order, whatever the other nodes do:
//   1. state OPT_CACHED: the cached masks are Transacted, stale or not (a failure keeps its Adds, gpu.go:153-175);
//      OPT_UNFIT: Trade fails on these rows, nothing binds; OPT_ABSENT: straight to 2;
//   2. Trade on the current rows, Transact, and again, until Trade fails.
// The row is a copy: the caller's is not written.  At most `limit` binds (successful or failed) are made; `capped`
// says the node still had an option when the limit stopped it.
// ---------------------------------------------------------------------------------------------
struct Headroom { int ok, failed, capped; };

template <int G, class R>
EGS_HD Headroom headroom_node(const int (&c0)[G], const int (&m0)[G], int mem_total, const R &r, bool single,
                              int policy, int state, PackedT<G, R::NC> masks, int limit) {
  Headroom h = {0, 0, 0};
  if (state == OPT_UNFIT) return h;
  int c[G], m[G];
#pragma unroll
  for (int g = 0; g < G; g++) { c[g] = c0[g]; m[g] = m0[g]; }
  int score;
  bool have = state == OPT_CACHED || trade_any(c, m, mem_total, r, single, policy, score, masks);
  while (have) {
    if (h.ok + h.failed >= limit) { h.capped = 1; break; }
    if (transact_row<G>(c, m, mem_total, r, masks)) h.ok++; else h.failed++;
    have = trade_any(c, m, mem_total, r, single, policy, score, masks);
  }
  return h;
}

// One AddPod / ForgetPod row update with the option rebuilt from annotations (allocate.go:75-93): explicit index
// lists; a fractional container uses its first index only.  A whole-GPU container lists up to G indices.
template <int G>
struct ApplyOp { int node, cancel; ReqW req; int n_idx[EGS_CA]; int8_t idx[EGS_CA][G]; };

// The row update of a mutation record (egs_mutation, already validated) in the device's form: cancel 1 is ForgetPod's
// Cancel, 0 AddPod's Transact.  Host code: the mutation stream and the eviction what-if build their ops with it.
template <int G>
inline ApplyOp<G> apply_op_of(const egs_mutation &m, int cancel) {
  ApplyOp<G> o = {};
  o.node = m.node_id; o.cancel = cancel; o.req = make_req<ReqW>(m.n_containers, m.units);
  for (int c = 0; c < m.n_containers; c++) {
    o.n_idx[c] = m.n_idx[c];
    for (int j = 0; j < m.n_idx[c]; j++) o.idx[c][j] = m.idx[c][j];
  }
  return o;
}

// The update on the node's rows (one thread): Cancel (gpu.go:177-191, GPU.Sub gpu.go:41-49: a whole-GPU container
// puts its GPUs back at their totals) or Transact (gpu.go:153-175, CanAllocate + Add: the first failure stops the op,
// no rollback).  Returns false when a Transact stopped.
template <int G>
EGS_HD bool apply_op(int32_t *c, int32_t *m, int mt, const ApplyOp<G> &op) {
  for (int i = 0; i < op.req.C; i++) {
    const bool whole = op.req.cnt[i] > 0;
    const int lim = whole ? op.n_idx[i] : (op.n_idx[i] > 0 ? 1 : 0);
    for (int j = 0; j < lim; j++) {
      const int g = op.idx[i][j];
      if (op.cancel) {
        if (whole) { c[g] = EGS_CORE_PER_GPU; m[g] = mt; } else { c[g] += op.req.core[i]; m[g] += op.req.mem[i]; }
      } else if (whole) {
        if (!(c[g] == EGS_CORE_PER_GPU && m[g] == mt)) return false;
        c[g] = 0; m[g] = 0;
      } else {
        if (!(c[g] >= op.req.core[i] && m[g] >= op.req.mem[i])) return false;
        c[g] -= op.req.core[i]; m[g] -= op.req.mem[i];
      }
    }
  }
  return true;
}

// ---------------------------------------------------------------------------------------------
// Eviction what-if of one node (egs_evict_fit): would a pending pod fit on the node once its victims are gone?
// ForgetPod (node.go:129-140) changes only the node's rows and podsMap, not its option entries, and Assume / Score /
// Allocate (node.go:61-104) read only those rows and the node's entry for the shape, so the answer is the node's own:
//   1. the GPUs.Cancel of every victim that applies (the host's podsMap decisions: ops[0 .. n_ops)), on a copy of
//      the row;
//   2. the option: the cached one, stale or not (ForgetPod keeps it and Assume returns it, node.go:64-66); none when
//      the entry says "known not to fit" and no victim applied (the rows are those that memo was taken on); else
//      Trade on the freed row;
//   3. the bind: Transact of the option's masks on the freed row (gpu.go:153-175).
// On entry score / masks hold the cached option when state is OPT_CACHED.  Returns EGS_ERR_NOFIT (score and masks 0),
// EGS_OK, or EGS_ERR_TRANSACT (masks 0, score the option's).
// ---------------------------------------------------------------------------------------------
template <int G, class R>
EGS_HD int evict_node(const int (&c0)[G], const int (&m0)[G], int mem_total, const R &r, bool single, int policy,
                      int state, const ApplyOp<G> *ops, int n_ops, int &score, PackedT<G, R::NC> &masks) {
  int c[G], m[G];
#pragma unroll
  for (int g = 0; g < G; g++) { c[g] = c0[g]; m[g] = m0[g]; }
  for (int o = 0; o < n_ops; o++) apply_op<G>(c, m, mem_total, ops[o]);
  const bool have = state == OPT_CACHED ||
                    ((state != OPT_UNFIT || n_ops > 0) && trade_any(c, m, mem_total, r, single, policy, score, masks));
  if (!have) { score = 0; masks = 0; return EGS_ERR_NOFIT; }
  if (transact_row<G>(c, m, mem_total, r, masks)) return EGS_OK;
  masks = 0;
  return EGS_ERR_TRANSACT;
}
