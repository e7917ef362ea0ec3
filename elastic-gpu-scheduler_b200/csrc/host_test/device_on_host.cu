// device_on_host.cu -- the kernels' integer arithmetic (egs_device.cuh: Trade fast path, general Trade,
// Transact, the AddPod / ForgetPod row update) compiled for the HOST, so the CPU test suite can check the very
// source the GPU runs against the oracle (tests/test_device_arith_host.py).  Not part of libegs.
#include "../egs_device.cuh"

#include <vector>

template <int G>
static void rows(const int32_t *core, const int32_t *mem, int (&c)[G], int (&m)[G]) {
  for (int g = 0; g < G; g++) { c[g] = core[g]; m[g] = mem[g]; }
}

// The G-wide entry points below: rows of G cells, masks packed G bits per container.
template <int G>
static int trade_w(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                   int path, int32_t *score, PackedT<G> *masks) {
  int c[G], m[G];
  rows(core, mem, c, m);
  const Req r = make_req(C, units);
  const bool single = path == 0 && req_is_single(r);
  int sc = 0; PackedT<G> mk = 0;
  const bool ok = trade_any(c, m, mem_total, r, single, policy, sc, mk);
  *score = sc; *masks = mk;
  return ok ? 1 : 0;
}
template <int G>
static int apply_w(int32_t *core, int32_t *mem, int mem_total, int C, const egs_unit *units, const int32_t *n_idx,
                   const int32_t *idx, int cancel) {
  ApplyOp<G> op = {};
  op.cancel = cancel; op.req = make_req<ReqW>(C, units);
  for (int c = 0; c < C; c++) {
    op.n_idx[c] = n_idx[c];
    for (int j = 0; j < n_idx[c]; j++) op.idx[c][j] = (int8_t)idx[c * G + j];
  }
  return apply_op(core, mem, mem_total, op) ? 1 : 0;
}

// headroom_node (k_headroom's per-node loop) at geometry (G, NP) = (8, 4), (16, 4) or (8, 8): rows of G cells, the
// option entry's state (OPT_*) and packed masks, the kernels' Trade dispatch.  out = {ok, failed, capped}.
template <int G, int NP>
static void headroom_w(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                       int state, uint64_t masks, int limit, int32_t *out) {
  int c[G], m[G];
  rows(core, mem, c, m);
  const ReqOf<NP> r = make_req<ReqOf<NP>>(C, units);
  const bool single = C == 1 && r.cnt[0] == 0 && r.core[0] >= 0 && r.mem[0] >= 0;
  const Headroom h = headroom_node(c, m, mem_total, r, single, policy, state, (PackedT<G, NP>)masks, limit);
  out[0] = h.ok; out[1] = h.failed; out[2] = h.capped;
}

// evict_node (k_evict's per-node answer) at geometry (G, NP): rows of G cells, the option entry's state, score and
// packed masks, and the victims that apply as egs_mutation records (converted as egs_evict_fit converts them).
// out = {status, score}; *masks the masks of a successful bind.
template <int G, int NP>
static void evict_w(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                    int state, int score, uint64_t *masks, int n_victims, const egs_mutation *victims, int32_t *out) {
  int c[G], m[G];
  rows(core, mem, c, m);
  const ReqOf<NP> r = make_req<ReqOf<NP>>(C, units);
  const bool single = C == 1 && r.cnt[0] == 0 && r.core[0] >= 0 && r.mem[0] >= 0;
  std::vector<ApplyOp<G>> ops;
  for (int k = 0; k < n_victims; k++) ops.push_back(apply_op_of<G>(victims[k], 1));
  PackedT<G, NP> mk = (PackedT<G, NP>)*masks;
  out[0] = evict_node(c, m, mem_total, r, single, policy, state, ops.data(), n_victims, score, mk);
  out[1] = score; *masks = mk;
}

extern "C" {
// path: 0 = the dispatch the kernels use (fast path when req_is_single), 1 = always the general DFS
int egsdh_trade(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                int path, int32_t *score, uint32_t *masks) {
  return trade_w<EGS_G>(core, mem, mem_total, C, units, policy, path, score, masks);
}
// the same on a 16-wide row (a wide handle): masks are 4 x u16
int egsdh_trade16(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                  int path, int32_t *score, uint64_t *masks) {
  return trade_w<16>(core, mem, mem_total, C, units, policy, path, score, masks);
}
// the leaf-parallel Trade the resolver runs across a warp, serially: max over (score, leaf index)
int egsdh_trade_leaves(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                       int32_t *score, uint32_t *masks) {
  int c[EGS_G], m[EGS_G];
  rows(core, mem, c, m);
  const Req r = make_req(C, units);
  int bits, nbranch, nleaf;
  trade_leaf_space(c, r, bits, nbranch, nleaf);
  long long best = -1; uint32_t bm = 0;
  for (int leaf = 0; leaf < nleaf; leaf++) {
    uint32_t mk = 0;
    const int sc = trade_leaf_eval(c, m, mem_total, r, policy, bits, nbranch, leaf, mk);
    if (sc < 0) continue;
    const long long key = ((long long)sc << 20) | leaf;
    if (key > best) { best = key; bm = mk; }
  }
  if (best < 0) return 0;
  *score = (int32_t)(best >> 20); *masks = bm;
  return 1;
}
// the resolver's one-GPU-per-lane single-container Trade (trade_lane_key), serially: max over the lanes gl = 0..7,
// score and mask decoded from the winning key as the resolver does
int egsdh_trade_lanes(const int32_t *core, const int32_t *mem, int rq_core, int rq_mem, int policy, int32_t *score,
                      uint32_t *masks) {
  int c[EGS_G], m[EGS_G];
  rows(core, mem, c, m);
  int bk = -1;
  for (int gl = 0; gl < EGS_G; gl++) { const int k = trade_lane_key(c, m, gl, rq_core, rq_mem, policy); bk = k > bk ? k : bk; }
  if (bk < 0) return 0;
  *score = policy == EGS_BINPACK ? (bk >> 3) * 100 : 0; *masks = 1u << (bk & 7);
  return 1;
}
int egsdh_transact(int32_t *core, int32_t *mem, int mem_total, int C, const egs_unit *units, uint32_t masks) {
  const Req r = make_req(C, units);
  return transact_row<EGS_G>(core, mem, mem_total, r, masks) ? 1 : 0;
}
int egsdh_transact16(int32_t *core, int32_t *mem, int mem_total, int C, const egs_unit *units, uint64_t masks) {
  const Req r = make_req(C, units);
  return transact_row<16>(core, mem, mem_total, r, masks) ? 1 : 0;
}
// apply_op (k_apply / k_apply_many) on one node's rows: C <= EGS_MAX_CONTAINERS_APPLY containers, container c's
// GPU indices in idx[c*EGS_MAX_GPUS .. + n_idx[c])
int egsdh_apply(int32_t *core, int32_t *mem, int mem_total, int C, const egs_unit *units, const int32_t *n_idx,
                const int32_t *idx, int cancel) {
  return apply_w<EGS_G>(core, mem, mem_total, C, units, n_idx, idx, cancel);
}
// the same on a 16-wide row: container c's indices in idx[c*16 .. + n_idx[c]), up to 16
int egsdh_apply16(int32_t *core, int32_t *mem, int mem_total, int C, const egs_unit *units, const int32_t *n_idx,
                  const int32_t *idx, int cancel) {
  return apply_w<16>(core, mem, mem_total, C, units, n_idx, idx, cancel);
}
// The general DFS Trade at geometry (8, 8) -- a sidecar handle's one-thread Trade -- for C <= 8 containers: masks
// are 8 x u8.  path as in egsdh_trade.
int egsdh_trade8c(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                  int path, int32_t *score, uint64_t *masks) {
  int c[EGS_G], m[EGS_G];
  rows(core, mem, c, m);
  const ReqW r = make_req<ReqW>(C, units);
  const bool single = path == 0 && C == 1 && r.cnt[0] == 0 && r.core[0] >= 0 && r.mem[0] >= 0;
  int sc = 0; PackedT<EGS_G, EGS_CA> mk = 0;
  const bool ok = trade_any(c, m, mem_total, r, single, policy, sc, mk);
  *score = sc; *masks = mk;
  return ok ? 1 : 0;
}
// The leaf-split Trade's reduction (k_trade_leaves + k_trade_commit) for C <= 8 containers, serially: the leaf space
// of digit width `bits` is cut into chunks of `chunk` leaves, the chunks are walked in the order of a Fisher-Yates
// shuffle drawn from `seed`, each chunk in leaf order with the kernel's pruning, and the 64-bit keys are max-reduced;
// the winner is decoded as the commit decodes it.  *n_eval: leaves evaluated (pruned ones are not).
int egsdh_trade_split(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units, int policy,
                      int bits, int chunk, uint64_t seed, int32_t *score, uint64_t *masks, int64_t *n_eval) {
  int c[EGS_G], m[EGS_G];
  rows(core, mem, c, m);
  const ReqW r = make_req<ReqW>(C, units);
  int nbranch = 0;
  for (int i = 0; i < C; i++) nbranch += r.cnt[i] > 0 ? 0 : 1;
  const int nleaf = 1 << (bits * nbranch), nchunk = (nleaf + chunk - 1) / chunk;
  std::vector<int> order(nchunk);
  for (int k = 0; k < nchunk; k++) order[k] = k;
  for (int k = nchunk - 1; k > 0; k--) std::swap(order[k], order[mix64(seed ^ (uint64_t)k) % (uint64_t)(k + 1)]);
  unsigned long long best = 0; int64_t ev = 0;
  for (int k : order) {
    int leaf = k * chunk;
    const int end = std::min(leaf + chunk, nleaf);
    while (leaf < end) {
      uint64_t mk; int fail;
      const int s = trade_leaf_eval(c, m, mem_total, r, policy, bits, nbranch, leaf, mk, &fail);
      ev++;
      if (s >= 0) {
        const unsigned long long key = ((unsigned long long)(uint32_t)s << 32) | (unsigned)(leaf + 1);
        best = std::max(best, key);
        leaf++;
      } else {
        leaf = trade_leaf_next(leaf, fail, bits, nbranch);
      }
    }
  }
  *n_eval = ev;
  if (!best) return 0;
  uint64_t mk = 0;
  trade_leaf_eval(c, m, mem_total, r, policy, bits, nbranch, (int)(uint32_t)best - 1, mk);
  *score = (int32_t)(best >> 32); *masks = mk;
  return 1;
}
// One leaf through both leaf evaluations: the resolver's (Req, 32-bit masks) and the leaf-split Trade's template (ReqW,
// 64-bit masks), for C <= EGS_MAX_CONTAINERS.  The two are separate definitions and must agree leaf for leaf.
void egsdh_leaf_eval_both(const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units,
                          int policy, int bits, int leaf, int32_t *s4, uint32_t *m4, int32_t *s8, uint64_t *m8) {
  int c[EGS_G], m[EGS_G];
  rows(core, mem, c, m);
  const Req r = make_req(C, units);
  const ReqW rw = make_req<ReqW>(C, units);
  int nbranch = 0;
  for (int i = 0; i < C; i++) nbranch += r.cnt[i] > 0 ? 0 : 1;
  uint32_t a = 0; uint64_t b = 0;
  *s4 = trade_leaf_eval(c, m, mem_total, r, policy, bits, nbranch, leaf, a);
  *s8 = trade_leaf_eval(c, m, mem_total, rw, policy, bits, nbranch, leaf, b);
  *m4 = *s4 >= 0 ? a : 0; *m8 = *s8 >= 0 ? b : 0;
}
// headroom_w at the geometry of a handle: g == 16 a wide handle, planes == 8 a sidecar handle
void egsdh_headroom(int g, int planes, const int32_t *core, const int32_t *mem, int mem_total, int C,
                    const egs_unit *units, int policy, int state, uint64_t masks, int limit, int32_t *out) {
  if (g == 16) headroom_w<16, EGS_C>(core, mem, mem_total, C, units, policy, state, masks, limit, out);
  else if (planes == EGS_CA) headroom_w<EGS_G, EGS_CA>(core, mem, mem_total, C, units, policy, state, masks, limit, out);
  else headroom_w<EGS_G, EGS_C>(core, mem, mem_total, C, units, policy, state, masks, limit, out);
}
// evict_w at the geometry of a handle: g == 16 a wide handle, planes == 8 a sidecar handle
void egsdh_evict(int g, int planes, const int32_t *core, const int32_t *mem, int mem_total, int C, const egs_unit *units,
                 int policy, int state, int score, uint64_t *masks, int n_victims, const egs_mutation *victims,
                 int32_t *out) {
  if (g == 16) evict_w<16, EGS_C>(core, mem, mem_total, C, units, policy, state, score, masks, n_victims, victims, out);
  else if (planes == EGS_CA) evict_w<EGS_G, EGS_CA>(core, mem, mem_total, C, units, policy, state, score, masks, n_victims, victims, out);
  else evict_w<EGS_G, EGS_C>(core, mem, mem_total, C, units, policy, state, score, masks, n_victims, victims, out);
}
int egsdh_is_single(int C, const egs_unit *units) { const Req r = make_req(C, units); return req_is_single(r) ? 1 : 0; }
unsigned long long egsdh_cand_key(int32_t score, uint32_t node) { return cand_key(score, node); }
unsigned long long egsdh_fit_term(uint32_t node) { return fit_term(node); }
unsigned long long egsdh_score_term(uint32_t node, int32_t score) { return score_term(node, score); }
}
