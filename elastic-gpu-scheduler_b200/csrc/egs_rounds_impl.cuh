// egs_rounds_impl.cuh -- host side of EGS_MODE_ROUNDS (included at the end of egs_api.cu).
#pragma once
#include <dlfcn.h>
#include <nccl.h>   // types only: the library is resolved at run time (see nccl_api)

// NCCL is NOT a link-time dependency: a process that also hosts PyTorch must end up with ONE
// libnccl (torch bundles its own, newer than the system one).  dlopen by soname returns the
// copy that is already mapped, else the system library.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
static NcclApi *nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api.ok ? &api : nullptr;
  tried = true;
  void *lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!lib) return nullptr;
  api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(lib, "ncclGetUniqueId");
  api.CommInitRank = (decltype(api.CommInitRank))dlsym(lib, "ncclCommInitRank");
  api.CommDestroy = (decltype(api.CommDestroy))dlsym(lib, "ncclCommDestroy");
  api.AllGather = (decltype(api.AllGather))dlsym(lib, "ncclAllGather");
  api.GetErrorString = (decltype(api.GetErrorString))dlsym(lib, "ncclGetErrorString");
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString;
  return api.ok ? &api : nullptr;
}

#define NCK(h, call)                                                                     \
  do {                                                                                   \
    ncclResult_t r_ = (call);                                                            \
    if (r_ != ncclSuccess) {                                                             \
      (h)->err = std::string(#call) + ": " + nccl_api()->GetErrorString(r_);                     \
      return EGS_ERR_COMM;                                                               \
    }                                                                                    \
  } while (0)

// The NCCL comm and the events; the buffers go with the handle.
static void rounds_free(RoundsState *r) {
  if (r->comm && nccl_api()) nccl_api()->CommDestroy((ncclComm_t)r->comm);
  if (r->ev_ready) cudaEventDestroy(r->ev_ready);
  if (r->ev_copied) cudaEventDestroy(r->ev_copied);
}

static int rounds_comm_unique_id(uint8_t out_id[128]) {
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  ncclUniqueId id;
  if (!nccl_api() || nccl_api()->GetUniqueId(&id) != ncclSuccess) return EGS_ERR_COMM;
  memcpy(out_id, &id, 128);
  return EGS_OK;
}

static int rounds_comm_init(egs_handle *h, const uint8_t id[128]) {
  if (h->world < 2) return fail(h, EGS_ERR_BAD_ARG, "egs_shard_set first");
  if (!nccl_api()) return fail(h, EGS_ERR_COMM, "libnccl.so.2 not found");
  if (h->rounds.comm) { nccl_api()->CommDestroy((ncclComm_t)h->rounds.comm); h->rounds.comm = nullptr; }
  ncclUniqueId uid; memcpy(&uid, id, 128);
  ncclComm_t comm;
  NCK(h, nccl_api()->CommInitRank(&comm, h->world, uid, h->rank));
  h->rounds.comm = comm;
  return EGS_OK;
}


// In-process shard group over `world` handles (rank r = handles[r], each already egs_shard_set(r, world)).
static int rounds_comm_init_local(egs_handle **handles, int world) {
  if (!handles || world < 2 || world > RD) return EGS_ERR_BAD_ARG;
  auto G = std::make_shared<LocalGroup>();
  G->world = world;
  for (int r = 0; r < world; r++) {
    egs_handle *h = handles[r];
    if (!h || h->world != world || h->rank != r) return EGS_ERR_BAD_ARG;
    G->members.push_back(h);
  }
  for (int r = 0; r < world; r++) {
    egs_handle *h = handles[r];
    std::lock_guard<std::mutex> lk(h->mu);
    cudaSetDevice(h->device);
    if (!h->rounds.ev_ready) {
      CK(h, cudaEventCreateWithFlags(&h->rounds.ev_ready, cudaEventDisableTiming));
      CK(h, cudaEventCreateWithFlags(&h->rounds.ev_copied, cudaEventDisableTiming));
    }
    h->rounds.local = G;
    h->rounds.copied = false;                                   // no peer of the new group has copied anything yet
  }
  return EGS_OK;
}

// k_select grid: enough warps for one 128-node chunk each, at most two CTAs per SM (every CTA then runs in one wave)
static int select_grid(const egs_handle *h) {
  const int chunks = (h->hi - h->lo + 127) / 128;
  return std::max(1, std::min((chunks + SEL_WARPS - 1) / SEL_WARPS, 2 * h->n_sm));
}

static int rounds_ensure(egs_handle *h, int P, const BufLayout &L) {
  RoundsState &R = h->rounds;
  if (!R.d_ctl) {
    CK(h, grow(h->stream, false, to(R.d_ctl, 1), to(R.h_ctl, 1), to(R.d_rd, 1), to(R.h_rd, 1)));
    for (int ns : {MwInst16::NS, MwInst32::NS, MwInst96::NS})
      CK(h, mw_dispatch(ns, [](auto i) {
        return cudaFuncSetAttribute(k_resolve_mw<decltype(i)>, cudaFuncAttributeMaxDynamicSharedMemorySize, MW_SMEM_MAX);
      }));
  }
  const size_t need = (size_t)L.bytes * RD;
  if (need > R.d_bufs.cap()) {
    CK(h, grow(h->stream, false, to(R.d_bufs, need)));
    CK(h, cudaMemsetAsync(R.d_bufs, 0, need, h->stream));
  }
  const int grid = select_grid(h);
  if (grid > R.grid || L.nsc > R.cta_nsc) {
    const int g = std::max(grid, R.grid), n = std::max(L.nsc, R.cta_nsc);
    CK(h, grow(h->stream, false, to(R.d_cta_lists, (size_t)g * n * RK), to(R.d_cta_agg, (size_t)g * n)));
    R.grid = g; R.cta_nsc = n;
  }
  if ((size_t)P + 8 > R.d_pod_sidx.cap()) CK(h, grow(h->stream, false, to(R.d_pod_sidx, (size_t)P + 8)));
  const size_t ns = h->shapes.size(), old = R.d_obs.cap();
  if (ns > old) {                                               // the flags of the slots held so far are kept
    CK(h, grow(h->stream, true, to(R.d_obs, std::max(ns, (size_t)4096))));
    CK(h, cudaMemsetAsync(R.d_obs + old, 0, R.d_obs.cap() - old, h->stream));
  }
  return EGS_OK;
}

// Runs the batch; *n_done = pods resolved (== P unless an error stopped the loop).  Under a node set d_set the cold
// fill and k_select leave every excluded node alone; the resolver needs no change, since it only tracks list nodes.
static int batch_rounds(egs_handle *h, int P, const std::vector<int> &slots, PodOut out, int *n_done,
                        const uint64_t *d_set) {
  RoundsState &R = h->rounds;
  *n_done = 0;
  if (h->world > 1 && !R.comm && !R.local) return fail(h, EGS_ERR_COMM, "sharded handle without egs_comm_init");
  if (h->world > RD) return fail(h, EGS_ERR_BAD_ARG, "too many shards");

  // distinct shapes of the whole batch, in order of first appearance: when they fit one round set the set
  // is the same for every round, the round loop runs without the host (no per-round synchronisation)
  std::vector<int> batch_shapes;
  {
    std::vector<char> seen(h->shapes.size(), 0);
    for (int p = 0; p < P && (int)batch_shapes.size() <= RSMAX; p++)
      if (!seen[slots[p]]) { seen[slots[p]] = 1; batch_shapes.push_back(slots[p]); }
  }
  const bool one_set = (int)batch_shapes.size() <= RSMAX;
  const int ns_cfg = one_set ? (int)batch_shapes.size() : RSMAX;
  const int D = h->world;
  const MwGeometry geo = mw_geometry(ns_cfg, D);
  const BufLayout L = make_layout(ns_cfg, geo.rkm);
  // in-process group: the peers copy this rank's buffer on THEIR streams in every round, the last round of the
  // previous batch included, and this rank synchronised only its own stream since.  Everything that rewrites or
  // frees the buffer -- rounds_ensure's reallocation, every round's k_merge -- waits for those copies.
  auto wait_peers_copied = [&]() -> int {
    if (R.local && R.copied)
      for (egs_handle *peer : R.local->members) if (peer != h) CK(h, cudaStreamWaitEvent(h->stream, peer->rounds.ev_copied, 0));
    return EGS_OK;
  };
  TRY(wait_peers_copied());
  TRY(rounds_ensure(h, P, L));

  TableSet tb; tb.st = h->tables.st; tb.sc = h->tables.sc; tb.al = h->tables.al; tb.n_pad = (size_t)h->n_pad; tb.n_slots = (int)h->shapes.size();
  const int grid = select_grid(h);
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  if (h->timing) for (auto &e : ev) CK(h, cudaEventCreate(&e));

  // Cold shapes (option table still all-absent, e.g. a fresh or restored scheduler): ONE full-evaluate launch
  // per shape over this shard's nodes fills the table (OPT_NEW / OPT_UNFIT) -- the HBM-roofline kernel,
  // N * (8G + 5 + C) bytes each; k_select then finds nothing left to Trade for them.  Under a node set the excluded
  // nodes stay OPT_ABSENT: k_select Trades them in a later batch whose set admits them.
  if (h->hi > h->lo) {
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int cold = 0;
    for (int slot : batch_shapes) {
      if (!one_set && cold >= RSMAX) break;
      if (!h->slot_cold[slot]) continue;
      if (!e0) { CK(h, cudaEventCreate(&e0)); CK(h, cudaEventCreate(&e1)); CK(h, cudaEventRecord(e0, h->stream)); }
      const Shape &sh = h->shapes[slot];
      EvalArgs ea;
      ea.core = h->d_core; ea.mem = h->d_mem; ea.mem_total = h->d_mem_total; ea.lo = h->lo; ea.n = h->hi - h->lo;
      ea.policy = h->policy; ea.req = make_req(sh.C, sh.u);
      ea.fit = tb.st + (size_t)slot * tb.n_pad; ea.score = tb.sc + (size_t)slot * tb.n_pad;
      ea.gpu = tb.al + (size_t)slot * EGS_C * tb.n_pad; ea.plane = tb.n_pad; ea.v_fit = OPT_NEW; ea.v_unfit = OPT_UNFIT;
      const NodeSet set{d_set};
      if (is_single(sh.C, sh.u)) {
        if (d_set) k_evaluate_nodes<EGS_G, true, 2><<<(ea.n + 511) / 512, 256, 0, h->stream>>>(ea, set);
        else k_evaluate<EGS_G, true, 2><<<(ea.n + 511) / 512, 256, 0, h->stream>>>(ea);
      } else {
        if (d_set) k_evaluate_nodes<EGS_G, false, 1><<<(ea.n + 255) / 256, 256, 0, h->stream>>>(ea, set);
        else k_evaluate<EGS_G, false, 1><<<(ea.n + 255) / 256, 256, 0, h->stream>>>(ea);
      }
      cold++;
    }
    if (e0) {
      CK(h, cudaEventRecord(e1, h->stream));
      CK(h, cudaEventSynchronize(e1));
      float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
      h->k_launches[EGS_K_EVALUATE] += cold; h->k_ms[EGS_K_EVALUATE] += ms;
      cudaEventDestroy(e0); cudaEventDestroy(e1);
      CK(h, cudaGetLastError());
    }
  }
  for (int slot : batch_shapes) h->slot_cold[slot] = 0;
  for (int p = 0; p < P; p++) h->slot_cold[slots[p]] = 0;

  // ---- resolver geometry
  const int rke = geo.rke;
  const size_t smem = geo.smem;
  if (rke < 4) return fail(h, EGS_ERR_BAD_ARG, "rounds: shape set too large for the resolver's shared memory");
  const int nw = std::max(1, std::min(ns_cfg, MW_MAX_WARPS));

  SelectArgs sa; MergeArgs ma; MwArgs ra;
  sa.core = h->d_core; sa.mem = h->d_mem; sa.mem_total = h->d_mem_total;
  sa.lo = h->lo; sa.hi = h->hi; sa.policy = h->policy; sa.nsc = L.nsc; sa.rd = R.d_rd; sa.tb = tb; sa.obs_pending = R.d_obs;
  sa.cta_lists = R.d_cta_lists; sa.cta_agg = R.d_cta_agg; sa.ctl = R.d_ctl;
  ma.core = h->d_core; ma.mem = h->d_mem; ma.mem_total = h->d_mem_total; ma.rd = R.d_rd; ma.tb = tb;
  ma.obs_pending = R.d_obs; ma.cta_lists = R.d_cta_lists; ma.cta_agg = R.d_cta_agg; ma.n_cta = grid;
  ma.out = R.d_bufs + (size_t)h->rank * L.bytes; ma.L = L; ma.ctl = R.d_ctl;
  ra.core = h->d_core; ra.mem = h->d_mem; ra.lo = h->lo; ra.hi = h->hi; ra.policy = h->policy; ra.n_shards = D;
  ra.rd = R.d_rd; ra.tb = tb; ra.obs_pending = R.d_obs; ra.bufs = R.d_bufs; ra.L = L; ra.pod_sidx = R.d_pod_sidx;
  ra.p0 = -1; ra.p_limit = 0; ra.out = out; ra.ctl = R.d_ctl; ra.rke = rke; ra.nw = nw; ra.pre_h = geo.pre_h; ra.pre_cap = geo.pre_cap;

  int ns_round = ns_cfg;                                        // grid of k_merge
  auto launch_round = [&]() -> int {
    if (h->timing) CK(h, cudaEventRecord(ev[0], h->stream));
    if (d_set) k_select_nodes<<<grid, SEL_THREADS, 0, h->stream>>>(sa, NodeSet{d_set});
    else k_select<<<grid, SEL_THREADS, 0, h->stream>>>(sa);
    if (h->timing) CK(h, cudaEventRecord(ev[1], h->stream));
    TRY(wait_peers_copied());                                   // peers must have copied my previous buffer before k_merge rewrites it
    k_merge<<<ns_round, 256, 0, h->stream>>>(ma);
    if (h->world > 1 && R.local) {
      // in-process group: wait until no peer still reads my buffer of the previous round (enqueued BEFORE k_merge
      // overwrote it, see below), publish mine, copy theirs
      LocalGroup &G = *R.local;
      CK(h, cudaEventRecord(R.ev_ready, h->stream));
      if (!G.barrier()) return fail(h, EGS_ERR_COMM, "in-process shard group: a member did not arrive");   // all recorded ev_ready
      for (egs_handle *peer : G.members) {
        if (peer == h) continue;
        CK(h, cudaStreamWaitEvent(h->stream, peer->rounds.ev_ready, 0));
        CK(h, cudaMemcpyAsync(R.d_bufs + (size_t)peer->rank * L.bytes, peer->rounds.d_bufs + (size_t)peer->rank * L.bytes,
                              (size_t)L.bytes, cudaMemcpyDeviceToDevice, h->stream));
      }
      CK(h, cudaEventRecord(R.ev_copied, h->stream));
      if (!G.barrier()) return fail(h, EGS_ERR_COMM, "in-process shard group: a member did not arrive");   // all recorded ev_copied
      R.copied = true;
    } else if (h->world > 1)
      NCK(h, nccl_api()->AllGather(R.d_bufs + (size_t)h->rank * L.bytes, R.d_bufs, (size_t)L.bytes, ncclChar, (ncclComm_t)R.comm, h->stream));
    if (h->timing) CK(h, cudaEventRecord(ev[2], h->stream));
    mw_dispatch(ns_cfg, [&](auto i) { k_resolve_mw<decltype(i)><<<1, 32 * nw, smem, h->stream>>>(ra); });
    if (h->timing) CK(h, cudaEventRecord(ev[3], h->stream));
    h->k_launches[EGS_K_SELECT] += 1; h->k_launches[EGS_K_MERGE] += 1; h->k_launches[EGS_K_RESOLVE] += 1;
    return EGS_OK;
  };
  auto read_ctl = [&]() -> int {
    CK(h, cudaMemcpyAsync(R.h_ctl, R.d_ctl, sizeof(RoundCtl), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaGetLastError());
    if (h->timing) {
      float a = 0, b = 0, c = 0;
      cudaEventElapsedTime(&a, ev[0], ev[1]); cudaEventElapsedTime(&b, ev[1], ev[2]); cudaEventElapsedTime(&c, ev[2], ev[3]);
      h->k_ms[EGS_K_SELECT] += a; h->k_ms[EGS_K_MERGE] += b; h->k_ms[EGS_K_RESOLVE] += c;
    }
    return EGS_OK;
  };

  // staging: pod -> shape index, round descriptor, control block
  TRY(ensure_stage(h, (size_t)P + 8));
  CK(h, cudaStreamSynchronize(h->stream));
  uint8_t *h_sidx = (uint8_t *)h->h_stage.get();
  RoundCtl ctl0; memset(&ctl0, 0, sizeof ctl0);
  std::vector<int> set_idx(h->shapes.size(), -1);
  int rc = EGS_OK;
  int resolved = 0;

  if (one_set) {
    RoundDesc &rd = *R.h_rd; memset(&rd, 0, sizeof rd);
    rd.ns = ns_cfg;
    for (int q = 0; q < ns_cfg; q++) {
      rd.slot[q] = batch_shapes[q]; set_idx[batch_shapes[q]] = q;
      rd.reqs[q] = make_req(h->shapes[batch_shapes[q]].C, h->shapes[batch_shapes[q]].u);
    }
    for (int q = ns_cfg; q < RSMAX; q++) rd.slot[q] = -1;
    for (int p = 0; p < P; p++) h_sidx[p] = (uint8_t)set_idx[slots[p]];
    memset(h_sidx + P, 0xFF, 8);
    ctl0.next_p = 0; ctl0.p_end = P;
    *R.h_ctl = ctl0;
    CK(h, cudaMemcpyAsync(R.d_rd, R.h_rd, sizeof(RoundDesc), cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(R.d_pod_sidx, h_sidx, (size_t)P + 8, cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(R.d_ctl, R.h_ctl, sizeof(RoundCtl), cudaMemcpyHostToDevice, h->stream));
    // rounds are enqueued in chunks; finished batches make the remaining launches of a chunk return at once
    int chunk = h->timing ? 1 : 8;
    int launched = 0;
    while (true) {
      for (int r = 0; r < chunk; r++) { rc = launch_round(); if (rc != EGS_OK) break; }
      if (rc != EGS_OK) break;
      launched += chunk;
      rc = read_ctl();
      if (rc != EGS_OK) break;
      resolved = R.h_ctl->next_p;
      if (R.h_ctl->error) { rc = fail(h, EGS_ERR_CUDA, "rounds: resolver made no progress"); break; }
      if (resolved >= P) break;
      if (!h->timing) {
        const double per_round = std::max(1.0, (double)resolved / std::max(1, (int)R.h_ctl->rounds));
        chunk = (int)std::min(256.0, std::max(4.0, (P - resolved) / per_round * 1.05 + 2.0));
      }
    }
  } else {
    // more distinct shapes than one set holds: the host forms the set of every round (one synchronisation per round)
    int p0 = 0;
    while (p0 < P) {
      RoundDesc &rd = *R.h_rd; memset(&rd, 0, sizeof rd);
      std::fill(set_idx.begin(), set_idx.end(), -1);
      int n = 0, plim = p0;
      for (; plim < P; plim++) {
        const int slot = slots[plim];
        if (set_idx[slot] < 0) {
          if (n == RSMAX) break;
          set_idx[slot] = n; rd.slot[n] = slot; rd.reqs[n] = make_req(h->shapes[slot].C, h->shapes[slot].u); n++;
        }
        h_sidx[plim] = (uint8_t)set_idx[slot];
      }
      rd.ns = n; ns_round = n;
      for (int q = n; q < RSMAX; q++) rd.slot[q] = -1;
      memset(h_sidx + plim, 0xFF, 8);
      ctl0.next_p = p0; ctl0.p_end = plim; ctl0.rounds = 0;
      *R.h_ctl = ctl0;
      CK(h, cudaMemcpyAsync(R.d_rd, R.h_rd, sizeof(RoundDesc), cudaMemcpyHostToDevice, h->stream));
      const int a0 = p0 & ~3;
      CK(h, cudaMemcpyAsync(R.d_pod_sidx + a0, h_sidx + a0, (size_t)(plim - a0) + 8, cudaMemcpyHostToDevice, h->stream));
      CK(h, cudaMemcpyAsync(R.d_ctl, R.h_ctl, sizeof(RoundCtl), cudaMemcpyHostToDevice, h->stream));
      rc = launch_round(); if (rc != EGS_OK) break;
      rc = read_ctl(); if (rc != EGS_OK) break;
      if (R.h_ctl->error || R.h_ctl->next_p <= p0) { rc = fail(h, EGS_ERR_CUDA, "rounds: resolver made no progress"); break; }
      R.rounds += 1; R.pods += R.h_ctl->next_p - p0; R.tracked += R.h_ctl->tracked;
      for (int i = 0; i < 4; i++) R.stops[i] += R.h_ctl->stops[i];
      // the resolver counts a round that reached p_end as "pod limit"; when pod plim < P is the first pod of a
      // shape outside this round's set, the round ended at its set boundary (egs.h: "shape outside the round set")
      if (R.h_ctl->next_p == plim && plim < P) { R.stops[0] -= 1; R.stops[1] += 1; }
      p0 = R.h_ctl->next_p;
      resolved = p0;
    }
  }
  if (one_set && R.h_ctl) {
    R.rounds += R.h_ctl->rounds; R.pods += R.h_ctl->pods; R.tracked += R.h_ctl->tracked;
    for (int i = 0; i < 4; i++) R.stops[i] += R.h_ctl->stops[i];
  }
  if (R.h_ctl) for (int i = 0; i < RPROF; i++) R.prof[i] += R.h_ctl->prof[i];
  if (h->timing) for (auto &e : ev) cudaEventDestroy(e);
  *n_done = std::min(resolved, P);
  // no OPT_NEW may outlive the batch -- also after an error, so that the handle stays consistent
  const int n = h->hi - h->lo;
  if (n > 0) k_rounds_finalize<<<(n + 255) / 256, 256, 0, h->stream>>>(tb, R.d_obs, h->lo, h->hi);   // a shard may be empty
  const int n_obs = (int)R.d_obs.cap();
  k_clear_u8<<<(n_obs + 255) / 256, 256, 0, h->stream>>>(R.d_obs, n_obs);
  if (rc != EGS_OK) return rc;
  CK(h, cudaGetLastError());
  return EGS_OK;
}
