// device_on_host.cu -- the kernels' integer arithmetic (egs_device.cuh: Trade fast path, general Trade,
// Transact, the AddPod / ForgetPod row update) compiled for the HOST, so the CPU test suite can check the very
// source the GPU runs against the oracle (tests/test_device_arith_host.py).  Not part of libegs.
#include "../egs_device.cuh"

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
int egsdh_is_single(int C, const egs_unit *units) { const Req r = make_req(C, units); return req_is_single(r) ? 1 : 0; }
unsigned long long egsdh_cand_key(int32_t score, uint32_t node) { return cand_key(score, node); }
unsigned long long egsdh_fit_term(uint32_t node) { return fit_term(node); }
unsigned long long egsdh_score_term(uint32_t node, int32_t score) { return score_term(node, score); }
}
