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
 *   opt_state[s][N] (u8), opt_score[s][N] (i32), opt_alloc[s][c][N] (GPU mask of container c,
 *   c < EGS_MASKS_PER_POD(c_max), EGS_MASK_BYTES(g_max) bytes).
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
#define EGS_MAX_CONTAINERS  4      /* containers per pod filter / score / bind take on a handle of egs_create */
#define EGS_MAX_CONTAINERS_APPLY 8 /* containers per pod AddPod / ForgetPod / replay account (sidecars count), and
                                      the largest pod a sidecar handle (egs_create_ex, c_max > 4) schedules */
#define EGS_CORE_PER_GPU    100    /* utils.GPUCoreEachCard, pkg/utils/types.go:6          */
#define EGS_MAX_MEM_PER_GPU (1 << 25) /* int32 guard: Range/(k+1)*100 must fit int32 (Go int is 64-bit) */
#define EGS_MAX_CORE_LOAD   (1 << 20) /* bound for free_core values given to egs_state_load */

/* Layout of a handle created with `g_max` GPUs per node and pods of up to `c_max` containers (c_max ==
 * EGS_MAX_CONTAINERS for egs_create) -- the one rule every row and mask buffer below follows:
 *   EGS_ROW_WIDTH(g_max)     int32 cells per node row (egs_state_dump): 8, or 16 on a wide handle;
 *   EGS_MASK_BYTES(g_max)    bytes per GPU mask, little endian, bit g = GPU g: 1, or 2 on a wide handle;
 *   EGS_MASKS_PER_POD(c_max) GPU masks per pod / node: 4, or 8 on a sidecar handle.
 * Every GPU mask output (egs_bind, egs_option_peek, egs_option_dump and out_alloc_mask of the egs_schedule_batch*
 * calls) holds EGS_MASKS_PER_POD(c_max) masks per pod / node, of which the first n_containers are meaningful (the
 * rest read 0): element (p, c) starts at byte (p*EGS_MASKS_PER_POD(c_max) + c) * EGS_MASK_BYTES(g_max).  On a handle
 * of egs_create this is EGS_MAX_CONTAINERS masks per pod, of one u8 each for g_max <= 8, as always. */
#define EGS_ROW_WIDTH(g_max)  ((g_max) > EGS_MAX_GPUS ? EGS_MAX_GPUS_WIDE : EGS_MAX_GPUS)
#define EGS_MASK_BYTES(g_max) ((g_max) > EGS_MAX_GPUS ? 2 : 1)
#define EGS_MASKS_PER_POD(c_max) ((c_max) > EGS_MAX_CONTAINERS ? EGS_MAX_CONTAINERS_APPLY : EGS_MAX_CONTAINERS)

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
/* egs_create for pods of up to `c_max` containers, 1 <= c_max <= EGS_MAX_CONTAINERS_APPLY (else EGS_ERR_BAD_ARG).
 * c_max <= EGS_MAX_CONTAINERS gives the handle egs_create gives.  5 <= c_max <= 8 gives a "sidecar" handle: filter,
 * score, bind, peek and egs_option_dump take 1..c_max containers -- a container without a GPU request is the sentinel
 * unit {-1,-1,0} and Trade tries it on every GPU, as the reference does -- and every mask output holds 8 masks per
 * pod (EGS_MASKS_PER_POD).  Its limits, each refused with EGS_ERR_BAD_ARG and an egs_last_error text:
 *   - its batch engine is the per-pod engine: EGS_MODE_AUTO runs EGS_MODE_RESCAN, EGS_MODE_ROUNDS is refused
 *     and applies nothing (also no record of egs_schedule_batch_mut);
 *   - egs_shard_set is refused;
 *   - egs_profile_evaluate takes at most EGS_MAX_CONTAINERS containers.
 * g_max > EGS_MAX_GPUS together with c_max > EGS_MAX_CONTAINERS is refused (EGS_ERR_BAD_ARG, no handle).
 * egs_mutation and the accounting verbs are the same on every handle. */
int egs_create_ex(int policy, int max_nodes, int g_max, int c_max, int device, egs_handle **out);
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
 * handle, see egs_create), pods with at most EGS_MAX_CONTAINERS containers (EGS_MAX_CONTAINERS_APPLY on a sidecar
 * handle, see egs_create_ex), per-GPU memory units
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
 *   out_alloc_mask     mask (p, c) at byte (p*EGS_MASKS_PER_POD(c_max) + c) * EGS_MASK_BYTES(g_max)
 *   out_fit_count[p]   number of fit nodes
 *   out_fit_digest[p]  sum over fit nodes of egs_mix64(2*node+1)                       (mod 2^64)
 *   out_score_digest[p] sum over fit nodes of egs_mix64(2*node+2) * (2*(u64)(u32)score + 1)             (mod 2^64)
 * The digests are sums so that node shards compose by addition.
 *
 * uids: NULL lets the library number the pods itself (pods awaiting scheduling are unknown to every
 * podsMap); otherwise they must be pairwise distinct and not yet known (EGS_ERR_BAD_ARG).  A bind that
 * reaches NodeAllocator.Add records the uid in that node's podsMap even when Transact fails (node.go:150);
 * only a successful bind enters podMaps (scheduler.go:224) -- visible through egs_pod_known.
 * EGS_MODE_AUTO == EGS_MODE_ROUNDS on a handle of egs_create with g_max <= EGS_MAX_GPUS, EGS_MODE_RESCAN on a
 * wide or sidecar handle (which refuse EGS_MODE_ROUNDS).  Both modes produce identical outputs; RESCAN is the literal
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
 * EGS_MASKS_PER_POD(c_max) * EGS_MASK_BYTES(g_max) bytes, so d_out_alloc_mask must be aligned to that size (4 bytes,
 * or 8 on a wide or sidecar handle; cudaMalloc memory always is): EGS_ERR_BAD_ARG otherwise. */
int egs_schedule_batch_device(egs_handle *h, int mode, int n_pods, const int32_t *h_c_off,
                              const egs_unit *h_units,
                              int32_t *d_out_node, int32_t *d_out_status, uint8_t *d_out_alloc_mask,
                              int32_t *d_out_fit_count, uint64_t *d_out_fit_digest,
                              uint64_t *d_out_score_digest);

/* egs_schedule_batch with a candidate node set per pod: the node list kube-scheduler passes after its own predicates
 * (node selectors and affinity, taints, cordoned and NotReady nodes), as GPUUnitScheduler.Assume receives it
 * (scheduler.go:112-168).  `sets` holds n_sets >= 1 bitmaps of EGS_NODE_SET_WORDS(max_nodes) words each; bit n & 63
 * of word n >> 6 admits node n.  Pod p uses set pod_set[p] (pod_set NULL: every pod uses set 0).
 * Pod p is scheduled exactly as the reference schedules it when passed the nodes of its set in ascending id order:
 * only those are filtered (Traded and cached), the fit ones scored, the first maximal one bound.  A node outside the
 * pod's set is not Traded, its options (stale ones included), its "known not to fit" memos and its rows stay as they
 * are, it counts in neither out_fit_count nor a digest, and it cannot win.  An all-ones set gives what
 * egs_schedule_batch gives; an empty set gives EGS_ERR_NOFIT with fit count 0 and changes nothing.
 * Outputs, uids, modes and the per-handle limits are those of egs_schedule_batch (EGS_MODE_ROUNDS stays refused on a
 * wide or sidecar handle, EGS_MODE_RESCAN stays single-shard); on a sharded handle every rank passes the same full
 * bitmaps.  EGS_ERR_BAD_ARG, before anything is applied: n_sets < 1, sets NULL, pod_set[p] outside [0, n_sets), or
 * a bit set at or beyond max_nodes.
 * Each run of consecutive pods with the same pod_set value is one batch of its own, with the library-assigned uids
 * continuing across runs as in one batch; a run stopped by an error keeps what earlier runs applied.
 * Cost model: the set is read per node by the kernels that already read that node, so one set costs what
 * egs_schedule_batch costs (config 4 on one H100 80GB HBM3 at 700 W, one run each: 0.95 M decisions/s without a set,
 * 0.98 M with an all-ones set, 0.99 M with a 90 % set).  Every run boundary ends a batch -- a host synchronisation, the result copies, the upload of
 * the next set and at least one round of its own -- about 0.3-0.5 ms at config 4 on that card: two pools alternating
 * in runs of 10 000 / 1 000 / 100 / 10 pods give 0.96 M / 0.77 M / 0.16 M / 0.024 M decisions/s.  So order the pods
 * set by set where that keeps each pod's decision (INTEGRATION.md 3). */
#define EGS_NODE_SET_WORDS(max_nodes) (((max_nodes) + 63) / 64)
int egs_schedule_batch_nodes(egs_handle *h, int mode, int n_pods, const int32_t *c_off, const egs_unit *units,
                             const uint64_t *uids, int n_sets, const uint64_t *sets, const int32_t *pod_set,
                             int32_t *out_node, int32_t *out_status, uint8_t *out_alloc_mask,
                             int32_t *out_fit_count, uint64_t *out_fit_digest, uint64_t *out_score_digest);

/* ---- capacity: how many more pods of a shape the nodes take ------------------- */

/* Headroom: for each shape s and each node of [node0, node0+n), the number of pods of shape s the node would still
 * take if only pods of that shape arrived from now on, exactly as the scheduler would place them.
 *
 * Definition, and the equality that pins it: under a stream of pods of one shape, a node's Assume (node.go:61-73)
 * reads only its own rows and its own option entry, and a bind (node.go:87-104) writes only those; the driver rule
 * keeps binding while any node has an option.  So a dry run -- egs_checkpoint_save, egs_schedule_batch of K >= the
 * total identical pods, egs_checkpoint_rollback -- makes on every node the same sequence of binds in some order, and
 * this call counts that sequence node by node without running it:
 *   1. the shape's cached option on the node, if there is one, is Transacted first, even when stale (a stale option
 *      can fail its Transact; the Adds it made stay, gpu.go:153-175); a node whose entry says "known not to fit"
 *      (egs_option_dump state 2) takes nothing; a node without an entry starts at 2;
 *   2. Trade on the current rows under the handle's policy, Transact, and again, until Trade fails or `limit` binds
 *      (successful or failed) are made.
 * Per node, out_count[s*n + i] equals the EGS_OK pods of that dry run on node node0+i and out_failed[s*n + i] its
 * EGS_ERR_TRANSACT pods (at most 1, from a stale cached option); every pod after them is EGS_ERR_NOFIT.  With `set`
 * the equality holds against egs_schedule_batch_nodes with that set.
 * out_summary[s*4 + k]: k = 0 the sum of out_count, 1 the nodes with out_count > 0, 2 the sum of out_failed, 3 the
 * nodes stopped by `limit` that still had an option.  summary[3] > 0 means the answer is capped and summary[0] a
 * lower bound (a {0,0} container or a pod of sentinel units alone fits forever).
 *
 * Shape s has containers units[c_off[s] .. c_off[s+1]), checked like every request (up to c_max containers).
 * set: NULL for every node, else one bitmap of EGS_NODE_SET_WORDS(max_nodes) words in the egs_schedule_batch_nodes
 * layout; a node outside it counts 0 and is not read.  Any output may be NULL, not all three.
 * Read-only: rows, every option table, the pod maps, the next library-assigned uid and an open checkpoint stay as
 * they were; an unseen shape is interned as egs_option_dump interns it (its entries read "no entry", the state the
 * reference starts from).  A batch still in flight is finished first (stream order).
 * EGS_ERR_BAD_ARG with an egs_last_error text, nothing interned: n_shapes < 1, a shape of 0 or more than c_max
 * containers, node0 / n outside [0, max_nodes), a set bit at or beyond max_nodes, no output, limit < 1 or
 * limit > EGS_HEADROOM_MAX_LIMIT; on a sharded handle a range not inside the rank's egs_shard_range (its other rows
 * are stale after a sharded batch: each rank counts its own range and the host adds the ranks' summaries, no
 * collective runs); on a sidecar handle a shape the leaf-split kernels Trade (more than 2^12 leaves: not served by
 * this call).  A malformed unit returns what egs_filter returns for it.
 *
 * EGS_HEADROOM_MAX_LIMIT keeps every step of the per-node loop inside the int32 range the guards of egs_state_load
 * protect (DESIGN.md 1).  Rows start with free core <= 2^20 and free memory <= 2^25 per GPU, and only a sentinel
 * container raises a row, by 1 per bind: after L binds of a pod of up to 8 containers a GPU holds at most
 * 2^20 + 8L core and 2^25 + 8L memory, and the Trade of bind L+1 adds up to 8 more.  Binpack's score is
 * (max_mem + max_core - min_mem - min_core) / 2 / (k+1) * 100 with every row >= 0, so it stays below 2^31 while
 * (2^25 + 2^20) / 2 + 8(L+1) < 2^31 / 100, that is L + 1 < 521 666; L <= 2^18 leaves a factor of two. */
#define EGS_HEADROOM_MAX_LIMIT (1 << 18)
int egs_headroom(egs_handle *h, int n_shapes, const int32_t *c_off, const egs_unit *units, int node0, int n,
                 const uint64_t *set, int32_t limit, int32_t *out_count, int32_t *out_failed, int64_t *out_summary);

/* ---- eviction what-if: would a pending pod fit once a node's victims are gone ---- */

/* Eviction what-if: for each candidate node, whether the pending pod units[0 .. n_containers) would fit on it, and
 * bind with which masks, if the victims listed for that node were forgotten first -- kube-scheduler's preemption
 * question, asked of every candidate at once, with nothing changed.  Candidate node_ids[i] has the victims
 * victims[victim_off[i] .. victim_off[i+1]): EGS_MUT_FORGET records of that node, each with the units, index lists
 * and uid egs_pod_cancel would take (NewGPUOptionFromPod, allocate.go:75-93).  victim_off == NULL: no victims.
 *
 * Definition.  ForgetPod on node n (node.go:129-140) changes only n's rows and podsMap, not its option entries, and
 * Assume / Score / Allocate on n (node.go:61-104) read only n's rows and n's entry for the shape, so each node is
 * answered on its own, on a copy of its row:
 *   1. the GPUs.Cancel of every victim, in list order, that applies: its uid is in the node's podsMap and no earlier
 *      victim of the same list forgot it (the decision egs_pod_cancel takes, node.go:131);
 *   2. the option: the node's cached option of the shape, even when stale (ForgetPod keeps it, Assume returns it,
 *      node.go:64-66); none when the entry says "known not to fit" (egs_option_dump state 2) and no victim applied;
 *      else Trade on the freed row under the handle's policy;
 *   3. out_status[i]: EGS_ERR_NOFIT without an option, else the Transact of the option's masks on the freed row:
 *      EGS_OK, or EGS_ERR_TRANSACT when a stale cached option no longer fits (gpu.go:153-175);
 *      out_score[i]: the option's score (what egs_score returns), 0 for EGS_ERR_NOFIT;
 *      out_alloc_mask, element (i, c) at byte (i*EGS_MASKS_PER_POD(c_max) + c) * EGS_MASK_BYTES(g_max): the option's
 *      masks when out_status[i] is EGS_OK, else zeros (what egs_bind returns).
 * Per-node outputs follow the order of node_ids.
 *
 * Equality A, per node: egs_checkpoint_save; egs_pod_cancel of each victim of node_ids[i] in order;
 * egs_filter({node_ids[i]}), egs_score({node_ids[i]}) and, when it fits, egs_bind(node_ids[i], an unknown uid);
 * egs_checkpoint_rollback.  Filter says "no fit" exactly when out_status[i] is EGS_ERR_NOFIT; the score equals
 * out_score[i]; the bind's status and masks equal out_status[i] and the masks.
 * Equality B, all nodes at once: egs_checkpoint_save; egs_mutations_apply of every victim record of every candidate;
 * egs_schedule_batch_nodes of the one pending pod with the set of the candidate nodes; rollback.  With "fit" meaning
 * out_status != EGS_ERR_NOFIT, the batch's node is the lowest id among the fit nodes of maximal out_score (-1 when
 * none fits), its status and masks are that node's, its fit count is the number of fit nodes, and its digests are the
 * sums of the fit and score terms over the fit nodes -- whatever the order of node_ids.
 *
 * Read-only: rows, option tables, the pod maps, the next library-assigned uid and an open checkpoint stay as they
 * were; an unseen shape is interned as egs_option_dump interns it.  A batch still in flight is settled first.
 * Refused before anything is interned, with an egs_last_error text: n < 0, or n > 0 without node_ids or one of the
 * outputs (EGS_ERR_BAD_ARG); a node id check_node refuses (EGS_ERR_BAD_ARG out of range, EGS_ERR_NO_NODE not set);
 * a node id repeated (EGS_ERR_BAD_ARG); victim_off[0] != 0 or decreasing, or victims NULL with victim_off[n] > 0
 * (EGS_ERR_BAD_ARG); a victim of another kind or another node (EGS_ERR_BAD_ARG), or one egs_mutations_apply refuses
 * (its code: units, n_idx <= EGS_MAX_GPUS, indices below the node's GPU count); on a sidecar handle a pending shape the
 * leaf-split kernels Trade (EGS_ERR_BAD_ARG, as egs_headroom); on a sharded handle a node outside the rank's
 * egs_shard_range (EGS_ERR_BAD_ARG: an owner-only verb, like egs_filter).  A malformed pending unit returns what
 * egs_filter returns for it.  On a wide handle a whole-GPU victim of more than EGS_MAX_GPUS GPUs does not fit in a
 * record (as for egs_mutations_apply); the checkpoint recipe of equality A covers it. */
int egs_evict_fit(egs_handle *h, int n_containers, const egs_unit *units,
                  int n, const int32_t *node_ids, const int32_t *victim_off, const egs_mutation *victims,
                  int32_t *out_status, int32_t *out_score, uint8_t *out_alloc_mask);

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
