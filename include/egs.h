/*
 * egs.h -- C ABI of libegs, the H100-native GPU bin-packing scheduler core.
 *
 * Drop-in boundary for the hot path of elastic-ai/elastic-gpu-scheduler
 * (reference paths below are relative to the reference root):
 *
 *   pkg/scheduler/scheduler.go:30-39   ResourceScheduler interface  -> the verbs below
 *   pkg/scheduler/scheduler.go:112-168 GPUUnitScheduler.Assume      -> egs_filter
 *   pkg/scheduler/scheduler.go:170-184 GPUUnitScheduler.Score       -> egs_score
 *   pkg/scheduler/scheduler.go:186-199 GPUUnitScheduler.Bind        -> egs_bind
 *   pkg/scheduler/scheduler.go:229-267 AddPod / ForgetPod           -> egs_pod_apply / egs_pod_cancel
 *   pkg/scheduler/scheduler.go:269-281 KnownPod / ReleasedPod       -> egs_pod_known / egs_pod_released
 *   pkg/scheduler/scheduler.go:283-290 Status                       -> egs_state_dump
 *   pkg/scheduler/node.go:23-59        NewNodeAllocator             -> egs_node_set_allocatable / egs_node_set
 *
 * POD only: plain pointers and sizes, no Go pointers retained across calls
 * (cgo rule), no torch types.  Every entry point returns an egs_status and
 * never aborts the process.  A handle serialises its callers with an internal
 * mutex (the reference holds one global lock per verb, scheduler.go:113,171,187)
 * and calls cudaSetDevice on entry, so cgo thread-hopping is fine.
 *
 * The device state is an int32 SoA node/GPU cache:
 *   free_core[N][W], free_mem[N][W], mem_total[N]      W = EGS_ROW_WIDTH(g_max)
 * (CoreTotal == 100 for every GPU, pkg/utils/types.go:6) plus, per interned
 * request shape s, the per-node option cache of node.go:19
 *   opt_state[s][N] (u8), opt_score[s][N] (i32), opt_alloc[s][c][N] (GPU mask of container c, c < 4,
 *   EGS_MASK_BYTES(g_max) bytes).
 *
 * The INTEGRATION.md at the repo root shows the cgo binding.
 */
#ifndef EGS_H_
#define EGS_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EGS_MAX_GPUS        8      /* GPUs per node the SoA row of a handle with g_max <= 8 holds; width of egs_mutation */
#define EGS_MAX_GPUS_WIDE   16     /* widest node any handle takes (a "wide" handle: 9 <= g_max <= 16)                */
#define EGS_MAX_CONTAINERS  4      /* containers per pod the filter / score / bind path enumerates */
#define EGS_MAX_CONTAINERS_APPLY 8 /* containers per pod AddPod / ForgetPod / replay account (sidecars count) */
#define EGS_CORE_PER_GPU    100    /* utils.GPUCoreEachCard, pkg/utils/types.go:6          */
#define EGS_MAX_MEM_PER_GPU (1 << 25) /* int32 guard: Range/(k+1)*100 must fit int32 (Go int is 64-bit) */
#define EGS_MAX_CORE_LOAD   (1 << 20) /* bound for free_core values given to egs_state_load */

/* Layout of a handle created with `g_max` GPUs per node -- the one rule every row and mask buffer below follows:
 *   EGS_ROW_WIDTH(g_max)  int32 cells per node row (egs_state_dump): 8, or 16 on a wide handle;
 *   EGS_MASK_BYTES(g_max) bytes per GPU mask, little endian, bit g = GPU g: 1, or 2 on a wide handle.
 * Every GPU mask output (egs_bind, egs_option_peek, egs_option_dump and out_alloc_mask of the egs_schedule_batch*
 * calls) holds EGS_MAX_CONTAINERS masks per pod / node: element (p, c) starts at byte
 * (p*EGS_MAX_CONTAINERS + c) * EGS_MASK_BYTES(g_max).  For g_max <= 8 this is one u8 per container, as always. */
#define EGS_ROW_WIDTH(g_max)  ((g_max) > EGS_MAX_GPUS ? EGS_MAX_GPUS_WIDE : EGS_MAX_GPUS)
#define EGS_MASK_BYTES(g_max) ((g_max) > EGS_MAX_GPUS ? 2 : 1)

/* -priority flag, cmd/main.go:45-54 */
enum egs_policy { EGS_BINPACK = 0, EGS_SPREAD = 1 };

typedef enum egs_status {
  EGS_OK                 = 0,
  EGS_ERR_NOFIT          = 1,  /* "no enough resource to allocate"                 gpu.go:126 */
  EGS_ERR_NO_OPTION      = 2,  /* "cannot find option of GPU request %+v on %+v"   node.go:95 */
  EGS_ERR_TRANSACT       = 3,  /* "can't trade option %+v on %+v because ..."      gpu.go:160,168 */
  EGS_ERR_BAD_ARG        = 4,
  EGS_ERR_OVERFLOW_GUARD = 5,  /* value outside the int32-exact range              */
  EGS_ERR_CUDA           = 6,  /* see egs_last_error()                             */
  EGS_ERR_NO_GPU         = 7,  /* "no gpu available on node %s"                    node.go:29 */
  EGS_ERR_NO_NODE        = 8,  /* node id never set ("elastic gpu scheduler get node failed", scheduler.go:124) */
  EGS_ERR_PANIC          = 9,  /* the reference would panic here (nil option, node.go:84) */
  EGS_ERR_COMM           = 10  /* NCCL failure                                     */
} egs_status;

/* GPUUnit, gpu.go:9-13.  {-1,-1,0} is the NotNeedGPU sentinel (allocate.go:41-45). */
typedef struct egs_unit { int32_t core, mem, count; } egs_unit;

typedef struct egs_handle egs_handle;

/* ---- lifecycle ------------------------------------------------------------- */

/* One handle drives ONE device.  `g_max` <= EGS_MAX_GPUS_WIDE is the widest node it takes (17+: EGS_ERR_BAD_ARG).
 * A wide handle (g_max > EGS_MAX_GPUS) has 16-wide rows and 16-bit masks (EGS_ROW_WIDTH / EGS_MASK_BYTES) and
 * these limits, each refused with EGS_ERR_BAD_ARG and an egs_last_error text:
 *   - its batch engine is the per-pod engine: EGS_MODE_AUTO runs EGS_MODE_RESCAN, EGS_MODE_ROUNDS is refused
 *     and applies nothing (also no record of egs_schedule_batch_mut);
 *   - egs_shard_set is refused: the sharded engine is the rounds engine;
 *   - a mutation record still lists at most EGS_MAX_GPUS indices per container: a whole-GPU container of more
 *     than 8 GPUs goes through egs_pod_apply / egs_node_replay_pod / egs_pod_cancel, whose lists take up to 16. */
int egs_create(int policy, int max_nodes, int g_max, int device, egs_handle **out);
int egs_destroy(egs_handle *h);
const char *egs_last_error(egs_handle *h);
const char *egs_status_string(int status);        /* exact reference message where one exists */
/* NewGPURequest, allocate.go:35-58: (Requests[gpu-core], Requests[gpu-memory]) -> GPUUnit */
int egs_unit_from_requests(int64_t core, int64_t mem, egs_unit *out);

/* ---- node cache (R1) ------------------------------------------------------- */

/* node.go:24-40: G = core_allocatable/100 (0 -> EGS_ERR_NO_GPU), M = mem_allocatable/G,
 * every GPU starts {100, M}.  Drops the node's option cache and podsMap. */
int egs_node_set_allocatable(egs_handle *h, int node_id, int64_t core_allocatable, int64_t mem_allocatable);
int egs_node_set(egs_handle *h, int node_id, int gpu_count, int mem_total_per_gpu);
/* Overwrite the free rows of one node (synthetic prefill / restore). */
int egs_state_load(egs_handle *h, int node_id, const int32_t *free_core, const int32_t *free_mem);
/* Bulk form: nodes [node0, node0+n), every node `gpu_count` GPUs of `mem_total`;
 * free_core/free_mem are [n][gpu_count] row-major. */
int egs_state_load_bulk(egs_handle *h, int node0, int n, int gpu_count, int mem_total,
                        const int32_t *free_core, const int32_t *free_mem);
/* Status(), scheduler.go:283-290: rows of nodes [node0, node0+n) as [n][EGS_ROW_WIDTH(g_max)]
 * (absent GPUs read as INT32_MIN), gpu_count[n], mem_total[n]; any out pointer may be NULL. */
int egs_state_dump(egs_handle *h, int node0, int n, int32_t *free_core, int32_t *free_mem,
                   int32_t *gpu_count, int32_t *mem_total);

/* Device-side checkpoint of the rows, and its restore.  Restore also empties every option
 * cache and the pod maps: the state of a freshly restarted scheduler whose node cache was
 * rebuilt (scheduler.go:86-106).  Used by bench.py to start every step from the same cluster. */
int egs_state_snapshot(egs_handle *h);
int egs_state_restore(egs_handle *h);

/* Checkpoint of the COMPLETE scheduler state, for dry runs, all-or-nothing admission of a
 * pod group and what-if evictions (INTEGRATION §3).  Unlike egs_state_restore, which is a
 * restarted scheduler, a rollback is exact: every call made after it answers as it would
 * have answered at the save.  The state is
 *   - the rows, mem_total, and which nodes are set with how many GPUs;
 *   - the option cache of every shape interned at the save (cached options, stale ones
 *     included, and "does not fit" memos); shapes interned after the save are forgotten;
 *   - podsMap, podMaps and releasedPodMap (egs_pod_known / egs_pod_released);
 *   - the next library-assigned uid, so a dry run and the real run that follows it assign
 *     the same uids.
 * Not state: the egs_state_snapshot copy, profile counters and egs_rounds_stats,
 * egs_last_error, and the shard / communicator setup.
 * Batches still pending are settled at the save; a rollback discards whatever batch ran
 * after it.  Costs: two device copies of the rows and of the option tables in use, plus
 * host work proportional to the uid bookkeeping changed since the save.
 *
 * save: records the state, replacing an earlier checkpoint.
 * rollback: returns to it; the checkpoint stays, so several what-ifs can start from it.
 *   With no checkpoint: EGS_ERR_BAD_ARG (egs_last_error says so), nothing changes.
 * drop: forgets it and frees its memory; the current state stays.
 * egs_destroy frees a checkpoint and egs_shard_set drops it.  On a sharded handle every
 * rank issues the calls, as with every other call; no collective runs.  One checkpoint
 * per handle: they do not nest. */
int egs_checkpoint_save(egs_handle *h);
int egs_checkpoint_rollback(egs_handle *h);
int egs_checkpoint_drop(egs_handle *h);

/* ---- verbs (one pod at a time; host buffers) -------------------------------- */

/* Assume: for each candidate node (node_ids == NULL means 0..n-1) cache hit -> fit,
 * else Trade (gpu.go:65-129) and cache on success (node.go:61-73).  out_fit[i] in {0,1}. */
int egs_filter(egs_handle *h, int n, const int32_t *node_ids, int n_containers,
               const egs_unit *units, uint8_t *out_fit);
/* Score: cached option.Score per node (node.go:75-85); unknown node -> 0
 * (scheduler.go:176-179).  Returns EGS_ERR_PANIC if some node had no entry but fits. */
int egs_score(egs_handle *h, int n, const int32_t *node_ids, int n_containers,
              const egs_unit *units, int32_t *out_score);
/* Bind -> NodeAllocator.Allocate (node.go:87-104): consumes the cached option, Transact
 * without rollback (gpu.go:153-175).  out_alloc_mask mask c has bit g set when GPU g goes to
 * container c (Trade only ever yields ascending index lists, so the mask is lossless); EGS_MASK_BYTES per mask. */
int egs_bind(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
             uint64_t uid, uint8_t *out_alloc_mask);
/* Inspect the cached option of (node, request) without side effects (tests, Assume's GPUIDs). */
int egs_option_peek(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                    int32_t *out_valid, int32_t *out_score, uint8_t *out_alloc_mask);

/* Bulk form of egs_option_peek: the option cache (node.go:19 `allocated`) of one request on nodes
 * [node0, node0+n) -- the per-shape part of Status() / a checkpoint.  out_state[i]: 0 no entry, 1 entry
 * present (possibly stale), 2 no entry and the request is known not to fit the current rows;
 * out_score[i] / the mask (i, c) of out_alloc_mask are meaningful for state 1.  Any out may be NULL. */
int egs_option_dump(egs_handle *h, int n_containers, const egs_unit *units, int node0, int n,
                    uint8_t *out_state, int32_t *out_score, uint8_t *out_alloc_mask);

/* AddPod (scheduler.go:229-245 -> node.go:148-160 with the option rebuilt from the
 * annotations, allocate.go:75-93).  alloc_idx[alloc_off[c] .. alloc_off[c+1]) are the
 * GPU indices of container c in annotation order.  The three accounting verbs below (and the mutation records)
 * take pods of up to EGS_MAX_CONTAINERS_APPLY containers: a pod another scheduler placed -- sidecars included --
 * is subtracted from the node cache exactly like the reference does, also when this library could not have
 * scheduled it (filter / score / bind stop at EGS_MAX_CONTAINERS). */
int egs_pod_apply(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                  const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid);
/* NodeAllocator.Add(pod, nil) alone (node.go:148-160), as NewNodeAllocator replays the pods already
 * assumed on a node when it is first loaded (node.go:52-54): node-level podsMap + Transact, the
 * scheduler-level podMaps is not touched. */
int egs_node_replay_pod(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                        const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid);
/* ForgetPod (scheduler.go:247-267 -> node.go:129-140 -> gpu.go:177-191); node_id < 0 == empty NodeName. */
int egs_pod_cancel(egs_handle *h, int node_id, int n_containers, const egs_unit *units,
                   const int32_t *alloc_off, const int32_t *alloc_idx, uint64_t uid);
/* ---- mutation stream (controller.go:154-185,301-331: AddPod / ForgetPod arrive between scheduling verbs, under the
 * same lock) and bulk start-up replay (scheduler.go:86-106, node.go:52-54) ---------------------------------------- */
enum egs_mutation_kind { EGS_MUT_ADD = 0,      /* AddPod     == egs_pod_apply       */
                         EGS_MUT_FORGET = 1,   /* ForgetPod  == egs_pod_cancel (node_id < 0: empty NodeName) */
                         EGS_MUT_REPLAY = 2 }; /* NodeAllocator.Add at node load == egs_node_replay_pod */
typedef struct egs_mutation {
  int32_t kind, node_id, n_containers, pad;
  egs_unit units[EGS_MAX_CONTAINERS_APPLY];
  int8_t n_idx[EGS_MAX_CONTAINERS_APPLY];               /* GPU indices of container c in annotation order ...      */
  int8_t idx[EGS_MAX_CONTAINERS_APPLY][EGS_MAX_GPUS];   /* ... idx[c][0 .. n_idx[c])                                */
  uint64_t uid;
} egs_mutation;
/* Applies the records IN ORDER -- observably identical to issuing the single-pod verbs one by one -- with ONE kernel
 * launch: the podsMap / podMaps decisions are taken on the host in record order, the surviving row updates are grouped
 * by node (order kept inside a node) and one thread per touched node applies them.  10^5 assumed pods replay in one
 * launch.  Returns the first record's error (nothing applied) when a record is malformed. */
int egs_mutations_apply(egs_handle *h, int n, const egs_mutation *ops);
/* egs_schedule_batch with a mutation stream woven in: record j is applied right before pod mut_at[j] (mut_at ascending,
 * 0 <= mut_at[j] <= n_pods; equal positions keep record order) -- the interleaving the reference's single lock produces
 * when the informer delivers AddPod / ForgetPod between two scheduling cycles.  Outputs as egs_schedule_batch. */
int egs_schedule_batch_mut(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                           const uint64_t *uids, int n_mut, const int32_t *mut_at, const egs_mutation *muts,
                           int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                           int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest);

int egs_pod_known(egs_handle *h, uint64_t uid);      /* 1 / 0, scheduler.go:269-274 */
int egs_pod_released(egs_handle *h, uint64_t uid);   /* 1 / 0, scheduler.go:276-281 */

/* ---- batch decision loop (device resident) ---------------------------------- */

/* Limits of the device path: nodes with at most EGS_MAX_GPUS_WIDE GPUs (more than EGS_MAX_GPUS only on a wide
 * handle, see egs_create), pods with at most EGS_MAX_CONTAINERS containers, per-GPU memory units
 * <= EGS_MAX_MEM_PER_GPU (use MiB, not bytes).
 * Anything beyond is refused with EGS_ERR_BAD_ARG / EGS_ERR_OVERFLOW_GUARD -- never computed differently.
 *
 * Driver rule (SURVEY.md 8d), identical to kube-scheduler's filter -> prioritize ->
 * bind round trip with ties broken to the first node: for each pod in order, filter
 * all nodes in index order, score the fit ones, winner = first fit node with the
 * maximum score, bind it.  Pod p has containers units[c_off[p] .. c_off[p+1]).
 *
 * Outputs (host pointers, any may be NULL):
 *   out_node[p]        winner node id, -1 when no node fits
 *   out_status[p]      EGS_OK / EGS_ERR_NOFIT / EGS_ERR_TRANSACT
 *   out_alloc_mask     mask (p, c) at byte (p*EGS_MAX_CONTAINERS + c) * EGS_MASK_BYTES(g_max)
 *   out_fit_count[p]   number of fit nodes
 *   out_fit_digest[p]  sum over fit nodes of egs_mix64(2*node+1)                       (mod 2^64)
 *   out_score_digest[p] sum over fit nodes of egs_mix64(2*node+2) * (2*(u64)(u32)score + 1)             (mod 2^64)
 * The digests are sums so that node shards compose by addition.
 *
 * uids: NULL lets the library number the pods itself (pods awaiting scheduling are unknown to every
 * podsMap); otherwise they must be pairwise distinct and not yet known (EGS_ERR_BAD_ARG).  A bind that
 * reaches NodeAllocator.Add records the uid in that node's podsMap even when Transact fails (node.go:150);
 * only a successful bind enters podMaps (scheduler.go:224) -- visible through egs_pod_known.
 * EGS_MODE_AUTO == EGS_MODE_ROUNDS on a handle with g_max <= EGS_MAX_GPUS, EGS_MODE_RESCAN on a wide handle
 * (which refuses EGS_MODE_ROUNDS).  Both modes produce identical outputs; RESCAN is the literal
 * one-pass-per-pod form (single shard only), ROUNDS the fast exact form (DESIGN.md 3).
 */
enum egs_batch_mode {
  EGS_MODE_AUTO   = 0,
  EGS_MODE_RESCAN = 1,  /* one full pass over every candidate node per pod           */
  EGS_MODE_ROUNDS = 2   /* exact round-based form: select top candidates, resolve    */
};
int egs_schedule_batch(egs_handle *h, int mode, int n_pods, const int32_t *c_off,
                       const egs_unit *units, const uint64_t *uids,
                       int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                       int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest);

/* The same driver rule with the FULL per-pod vectors materialised for pods [0, vec_pods): out_vec_fit[p*N + n] in {0,1}
 * and out_vec_score[p*N + n] (0 for unfit nodes) over all N = max_nodes nodes in index order -- what Assume returns
 * as filteredNodes and priority.go:26-39 as the HostPriorityList.  Runs the one-pass-per-pod engine (EGS_MODE_RESCAN,
 * single shard); the six per-pod outputs are as in egs_schedule_batch. */
int egs_schedule_batch_vec(egs_handle *h, int n_pods, const int32_t *c_off, const egs_unit *units, const uint64_t *uids,
                           int vec_pods, uint8_t *out_vec_fit, int32_t *out_vec_score,
                           int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                           int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest);

/* Same loop with every buffer already in device memory (bench `value` leg):
 * d_* are device pointers on the handle's device, laid out as above.  Each pod's masks are stored as one word of
 * EGS_MAX_CONTAINERS * EGS_MASK_BYTES(g_max) bytes, so d_out_alloc_mask must be aligned to that size (4 bytes, or 8 on
 * a wide handle; cudaMalloc memory always is): EGS_ERR_BAD_ARG otherwise. */
int egs_schedule_batch_device(egs_handle *h, int mode, int n_pods, const int32_t *h_c_off,
                              const egs_unit *h_units,
                              int32_t *d_out_node, int32_t *d_out_status, uint8_t *d_out_alloc_mask,
                              int32_t *d_out_fit_count, uint64_t *d_out_fit_digest,
                              uint64_t *d_out_score_digest);

/* ---- node sharding over several GPUs (one handle per device) ----------------- */

/* This handle owns nodes [lo, hi) of the max_nodes id space; rank/world describe the
 * shard order (world <= 8).  Every rank issues the same node_set / state_load / batch calls with the
 * FULL cluster; the batch loop exchanges the per-shape candidate buffers with ncclAllGather once per
 * round and every rank returns identical per-pod outputs.  After a sharded batch a rank's rows and
 * option tables are current only for its own range, so the single-pod verbs and egs_state_dump must be
 * addressed to the owner of the node.  NCCL is resolved at run time with dlopen("libnccl.so.2").
 *
 * Which rank gets which call, so that every rank's view of its own range stays the unsharded one:
 *   - every rank, with the same arguments and in the same order: node loads (egs_node_set_allocatable,
 *     egs_node_set, egs_state_load, egs_state_load_bulk), the accounting verbs (egs_pod_apply,
 *     egs_node_replay_pod, egs_pod_cancel), mutation records (egs_mutations_apply), batches
 *     (egs_schedule_batch, egs_schedule_batch_mut, egs_schedule_batch_device), snapshot / restore and checkpoints;
 *   - the owner of the node (egs_shard_range) alone: egs_filter, egs_score, egs_bind, egs_option_peek,
 *     egs_option_dump and egs_state_dump, over node ids of its own range.
 * A bind's uid enters the owner's pod maps only (egs_pod_known / egs_pod_released of it are the owner's); the uids
 * of a batch and of accounting verbs and records enter every rank's. */
int egs_shard_set(egs_handle *h, int rank, int world);
/* The contiguous node range [lo, hi) egs_shard_set gives rank `rank` of `world` (pure host
 * arithmetic, no handle): boundaries are multiples of 128, the last shard ends at max_nodes. */
int egs_shard_range(int max_nodes, int rank, int world, int *lo, int *hi);
int egs_comm_unique_id(uint8_t out_id[128]);
int egs_comm_init(egs_handle *h, const uint8_t id[128]);
/* In-process shard group instead of NCCL: handles[r] is rank r of `world` (each after egs_shard_set(r, world)), all in
 * this process -- on one device or several.  The per-round exchange becomes device-to-device copies ordered by CUDA
 * events; each handle's batch call must then be issued from its own thread, all `world` of them concurrently (they
 * rendezvous once per round).  Same kernels and buffers as the NCCL path: a single-GPU box can run the sharded engine. */
int egs_comm_init_local(egs_handle **handles, int world);

/* ---- instrumentation --------------------------------------------------------- */

enum egs_kernel_id { EGS_K_EVALUATE = 0, EGS_K_PASS = 1, EGS_K_SELECT = 2, EGS_K_RESOLVE = 3, EGS_K_MERGE = 4, EGS_K_COUNT = 8 };
/* Full-evaluate kernel alone (every candidate node Traded, no cache shortcut): runs
 * `iters` launches over nodes [0,n) for one request and reports the mean launch time
 * measured with CUDA events on the launching stream.  Does not modify the option cache. */
int egs_profile_evaluate(egs_handle *h, int n_containers, const egs_unit *units, int iters,
                         int flush_l2, float *out_ms_per_launch);
/* Launch counters / accumulated event time per kernel since the last reset. */
int egs_profile_get(egs_handle *h, int kernel_id, int64_t *out_launches, double *out_ms);
int egs_profile_reset(egs_handle *h, int enable_timing);

/* Counters of the round-based loop since creation: [0] rounds, [1] pods resolved, [2] tracked
 * nodes (sum over rounds), [3..6] rounds stopped by: pod limit, shape outside the round set,
 * tracked table full, candidate list dry. */
int egs_rounds_stats(egs_handle *h, int64_t out[8]);

/* The CUDA stream (cudaStream_t) every kernel of this handle is launched on, so that callers
 * can bracket work with CUDA events on the launching stream. */
int egs_get_stream(egs_handle *h, void **out_stream);

/* splitmix64 output function used by the digests */
uint64_t egs_mix64(uint64_t x);

#ifdef __cplusplus
}
#endif
#endif /* EGS_H_ */
