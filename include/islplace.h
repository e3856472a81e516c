/*
 * islplace.h — C ABI of the H100-native MIG-slot placement engine (libislplace.so).
 *
 * This is the drop-in boundary for ONE path of project-codeflare/instaslice: the
 * controller's allocator.  Every entry point below names the reference interface
 * it replaces (paths relative to the reference tree, commit b34e86d):
 *
 *   internal/controller/instaslice_controller.go
 *     :240-262  InstasliceReconciler.findDeviceForASlice      -> isl_place_batch
 *     :303-384  getStartIndexFromPreparedState                -> isl_place_batch / isl_eval_starts
 *     :283-300  extractGpuProfile                             -> isl_profile.{size,gi,ci,cieng} (echoed by the host shim)
 *     :48-50, :436-453  AllocationPolicy / FirstFitPolicy     -> isl_config.policy (the Go hook itself stays in Go and
 *                                                                packs AllocationDetails from isl_result)
 *   api/v1alpha1/instaslice_types.go
 *     :23-34    Mig / Placement                               -> isl_profile
 *     :37-50    AllocationDetails {start,size,gpuUUID,...}    -> isl_result {gpu,start,size,status}
 *     :53-62    PreparedDetails, :65-72 InstasliceSpec        -> isl_load_inventory (occupancy bytes built by the host shim
 *                                                                exactly as :306-328 does)
 *
 * Plain C, fixed-width integers, caller-owned buffers, no exceptions across the
 * boundary, no torch types.  The Go side binds it with cgo (INTEGRATION.md); the
 * tests and bench bind it with ctypes.
 *
 * Data model
 *   - G GPUs in canonical order (node index ascending, GPU index ascending inside
 *     a node; the host supplies the order, SURVEY.md section 8c "Q6").
 *   - occupancy: one byte per GPU, bit i set = memory slice i busy  (the
 *     reference's [8]uint32 gpuAllocatedIndex, :306).
 *   - profile table: up to ISL_MAX_PROFILES rows {size, ordered legal starts},
 *     one row per Migplacement entry (first entry with a given name wins for the
 *     start search, :332-340).
 *   - a request names a profile row; the engine answers (gpu, start) or "none"
 *     with the reference's sentinel start 9 (:248, :343).
 *
 * Batch semantics (canonical; DESIGN.md "Semantics"): within one batch every FREE
 * is applied first, then ALLOC requests are resolved strictly in array order,
 * each one seeing every earlier commit — identical to calling the reference's
 * allocator once per pod in that order on the same inventory.
 */
#ifndef ISLPLACE_H
#define ISLPLACE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ISL_ABI_VERSION      1u
#define ISL_MAX_PROFILES     16u          /* NVML_GPU_INSTANCE_PROFILE_COUNT is 0x11 incl. gaps; the reference tables have <= 10 rows */
#define ISL_MAX_STARTS       8u
#define ISL_MAX_TABLES       8u           /* distinct per-node Migplacement tables in one cluster (heterogeneous GPU models) */
#define ISL_SLOTS            8u           /* :306  var gpuAllocatedIndex [8]uint32 */
#define ISL_START_NONE       9u           /* :248, :343  notValidIndex */
#define ISL_GPU_NONE         0xFFFFFFFFu
#define ISL_MAX_GPUS         (1u << 24)   /* candidate records pack (gpu << 8 | occ) */
#define ISL_PROFILE_UNKNOWN  0xFFu        /* request for a profile name that is in no Migplacement row */

/* return codes */
#define ISL_OK        0
#define ISL_EINVAL   -1     /* malformed argument / table (the reference would panic: SURVEY Q7) */
#define ISL_ENOMEM   -2
#define ISL_ECUDA    -3     /* see isl_last_cuda_error */
#define ISL_ESTATE   -4     /* call order: profiles and inventory must be loaded before placing */
#define ISL_ERANGE   -5     /* batch or inventory larger than the engine was created for */

/* isl_config.policy */
#define ISL_POLICY_FIRST_FIT 0u   /* the only policy the reference implements (:66-67, :436) */
#define ISL_POLICY_BEST_FIT  1u   /* extension, no reference counterpart (SURVEY 8a-ext); parity unpinned: among the GPUs where the profile has a
                                     legal start, the one with the fewest free slices; ties -> lowest canonical index */
#define ISL_POLICY_RIGHT_TO_LEFT 2u /* first-fit over the GPUs in DESCENDING canonical order (last node first, last GPU of a node first) — what the
                                     reference's RightToLeftPolicy stub (:464-469) names but never implemented; ISL_POLICY_FIRST_FIT is its
                                     LeftToRightPolicy (:456-461).  The start inside a GPU still follows the row order (reverse the rows for
                                     right-to-left starts as well) */
#define ISL_POLICY_MIN_FRAG  3u   /* extension (SURVEY 8a-ext "richer score"): among the feasible GPUs, the one where the placement makes the fewest
                                     (profile, start) pairs of the table infeasible; ties -> lowest canonical index */

/* isl_config.quirks — bit set = reproduce the reference bug exactly */
#define ISL_QUIRK_STRICT_BOUND 1u /* Q1: `value+size < 8` (:351,:360,:370) instead of <= 8 */
#define ISL_QUIRK_POW2_ONLY    2u /* Q2: only sizes 1,2,4,8 are ever placed (:346-378) */
#define ISL_QUIRKS_REF_EXACT   (ISL_QUIRK_STRICT_BOUND | ISL_QUIRK_POW2_ONLY)
#define ISL_QUIRKS_FIXED       0u

/* isl_request.op; any other value is treated as ISL_OP_NOOP (record status ISL_ST_NOOP) */
#define ISL_OP_ALLOC 0u
#define ISL_OP_FREE  1u
#define ISL_OP_NOOP  2u

/* isl_result.status */
#define ISL_ST_PLACED      0u
#define ISL_ST_NO_CAPACITY 1u   /* the reference's error "failed to find allocatable gpu" (:261) on every node */
#define ISL_ST_BAD_PROFILE 2u   /* profile index >= loaded rows (the reference also ends at :261) */
#define ISL_ST_FREED       3u
#define ISL_ST_BAD_SPAN    4u   /* FREE outside the inventory or start+size > 8 (the reference would panic, Q7) */
#define ISL_ST_NOOP        5u
#define ISL_ST_GANG_ABORTED 6u  /* placeable as far as it was tried, but another member of its gang was not: nothing of the gang was committed */

typedef struct isl_engine isl_engine;

typedef struct isl_config {
    uint32_t abi_version;   /* ISL_ABI_VERSION */
    uint32_t policy;        /* ISL_POLICY_* */
    uint32_t quirks;        /* ISL_QUIRK_* mask; ISL_QUIRKS_REF_EXACT for bit-exact parity */
    int32_t  device;        /* CUDA device ordinal; -1 = current device */
    uint32_t max_gpus;      /* capacity, <= ISL_MAX_GPUS */
    uint32_t max_batch;     /* capacity of one isl_place_batch call (requests) */
    uint32_t flags;         /* ISL_FLAG_* */
    uint32_t reserved;
} isl_config;

#define ISL_FLAG_TIMING 1u  /* record per-kernel CUDA-event timings (isl_get_stats) */
#define ISL_FLAG_NO_PIPELINE    2u  /* always resolve chunk after chunk with the single-chain path */
#define ISL_FLAG_NO_SMALL      16u  /* do not use the fused single-launch kernel for batches of <= 1024 requests (tests) */
#define ISL_FLAG_TRACE          8u  /* record per (chunk, segment) timestamps of the segment pipeline (isl_read_trace) */
#define ISL_FLAG_FORCE_PIPELINE 4u  /* use the segment pipeline even for a single chunk (tests) */
#define ISL_FLAG_ALL_NODES     32u  /* isl_place_batch reproduces the reference's missing `break` (:190-227, SURVEY Q5): a pod is allocated on EVERY
                                       node that has capacity (state effect); the record reports the first node.  One restricted pass per node —
                                       a compatibility mode for parity studies, not a fast path */

/* One Migplacement row (api/v1alpha1/instaslice_types.go:23-29).  `size` is
 * Placements[0].Size (:334); `starts` is [p.Start for p in Placements] in CRD
 * order (:335-337), duplicates removed by the shim (a repeated start can never
 * change the first hit). */
typedef struct isl_profile {
    uint8_t  size;
    uint8_t  n_starts;
    uint8_t  starts[ISL_MAX_STARTS];
    uint8_t  pad[2];
    int32_t  gi_profile_id;     /* Giprofileid     */
    int32_t  ci_profile_id;     /* CIProfileID     */
    int32_t  ci_eng_profile_id; /* CIEngProfileID  */
} isl_profile;                  /* 24 bytes */

/* 8 bytes.  ALLOC: `profile` = row index (or ISL_PROFILE_UNKNOWN), `handle` is
 * opaque to the engine (the shim's pod index).  FREE: `handle` = canonical GPU
 * index, `start`/`size` = the span being released (an Allocations entry removed
 * by the daemonset, instaslice_daemonset.go:261-263). */
typedef struct isl_request {
    uint32_t handle;
    uint8_t  profile;
    uint8_t  op;
    uint8_t  start;
    uint8_t  size;
} isl_request;

/* 8 bytes; the fields of AllocationDetails the allocator decides
 * (instaslice_types.go:39-42).  gpu == ISL_GPU_NONE and start == 9 when nothing fits. */
typedef struct isl_result {
    uint32_t gpu;
    uint8_t  start;
    uint8_t  size;
    uint16_t status;
} isl_result;

typedef struct isl_span {
    uint32_t gpu;
    uint8_t  start;
    uint8_t  size;
    uint16_t pad;
} isl_span;

typedef struct isl_stats {
    uint64_t batches;
    uint64_t requests;
    uint64_t placed;
    uint64_t no_capacity;
    uint64_t freed;
    uint64_t kernel_launches;      /* kernels launched by this engine since creation */
    uint64_t chain_steps;          /* accepted placements walked by the commit chain */
    uint64_t chain_gpus_visited;   /* candidate GPUs the chain looked at */
    uint64_t chain_jumps;          /* ballot skips over candidates that no pending profile fits */
    /* accumulated CUDA-event milliseconds (only with ISL_FLAG_TIMING) */
    double   ms_free;
    double   ms_partition;
    double   ms_sweep;
    double   ms_commit;
    double   ms_total;             /* first kernel start -> last kernel end, per batch, summed */
    uint64_t scan_placed;          /* placements committed by the parallel capacity scan (single-profile chunks), no chain */
    /* speculative rounds (isl_set_speculation): chunks resolved that way, rounds until their last inventory stage was certified
     * (summed over the chunks), segment simulations run by all stages together */
    uint64_t spec_chunks;
    uint64_t spec_rounds;
    uint64_t spec_sims;
} isl_stats;

/* ---- lifetime ---------------------------------------------------------- */
int  isl_create(const isl_config* cfg, isl_engine** out);
int  isl_destroy(isl_engine* e);
/* Run all engine work on an existing CUDA stream (cudaStream_t passed as void*),
 * e.g. torch's current stream so that torch.cuda.Event brackets it. NULL = engine-owned stream. */
int  isl_set_stream(isl_engine* e, void* cuda_stream);
/* Wait for everything isl_place_batch_device / _partitioned enqueued (those two only enqueue). */
int  isl_synchronize(isl_engine* e);

/* ---- tables and inventory --------------------------------------------- */
/* Replaces reading instaslice.Spec.Migplacement (:332-340, :288-298). Builds the
 * per-(profile, occupancy byte) first-start table on the device. */
int  isl_load_profiles(isl_engine* e, uint32_t n, const isl_profile* rows);
/* Heterogeneous cluster: every node publishes its OWN Migplacement (instaslice_daemonset.go:588-664), and the reference
 * looks a profile up in the table of the node it is scanning (:332-340).  rows[t * n_profiles + p] is the row of profile
 * NAME p in table t; n_starts == 0 = that table has no row of the name (the reference then finds nothing on such a node).
 * Requests name a profile NAME index.  isl_set_node_tables (after isl_load_inventory) says which table each node uses
 * (default: table 0).  Every policy takes per-node tables (the best-fit family groups the GPUs by (table, occupancy byte)). */
int  isl_load_profile_tables(isl_engine* e, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows);
int  isl_set_node_tables(isl_engine* e, uint32_t n_nodes, const uint8_t* table_of_node);
/* Replaces the occupancy rebuild (:306-328) for every GPU of every node.
 * node_off has n_nodes+1 entries (node i owns GPUs [node_off[i], node_off[i+1]));
 * occ has node_off[n_nodes] bytes.  This is also "resume": the CR is the checkpoint. */
int  isl_load_inventory(isl_engine* e, uint32_t n_nodes, const uint32_t* node_off, const uint8_t* occ);
int  isl_read_occupancy(isl_engine* e, uint8_t* out /* G bytes */);
/* Incremental sync: overwrite the occupancy bytes of canonical GPUs [first_gpu, first_gpu + n) — what the shim does
 * when ONE Instaslice object changed (an Allocations / Prepared entry appeared or disappeared) instead of re-listing
 * every node (the reference deep-copies the whole list on every reconcile, :85). */
int  isl_write_occupancy(isl_engine* e, uint32_t first_gpu, uint32_t n, const uint8_t* occ);
/* What-if queries (defragmentation planning, SURVEY 8f-4): isl_snapshot_occupancy keeps a device-side copy of the whole
 * occupancy, any number of isl_place_* / isl_free_batch calls then run against the live state, isl_restore_occupancy puts the
 * snapshot back (a 1-byte-per-GPU device copy, no host round trip).  ISL_ESTATE if there is no inventory / no snapshot. */
int  isl_snapshot_occupancy(isl_engine* e);
int  isl_restore_occupancy(isl_engine* e);
/* cap[p] (ISL_MAX_PROFILES entries) = how many more pods of profile p ALONE the inventory (the engine's partition) could still take:
 * the sum over GPUs of the placements the start search (:343-383) would grant in a row.  A fragmentation measure per profile. */
int  isl_capacity(isl_engine* e, uint64_t* cap);
/* The what-if QUERY: resolve `plan` (FREEs and ALLOCs, batch semantics) against the live occupancy, report what fits (`out`) and the
 * per-profile capacity before and after (either may be NULL), then put the live state back — all under one engine lock, so no other
 * caller ever sees the hypothetical state.  "If these slices were released and these pods arrived: what fits, and what is left?"
 * (A snapshot taken with isl_snapshot_occupancy is invalidated by this call.) */
int  isl_what_if(isl_engine* e, uint32_t n, const isl_request* plan, isl_result* out, uint64_t* cap_before, uint64_t* cap_after);
uint32_t isl_num_gpus(const isl_engine* e);
/* node that owns canonical GPU index `gpu` (binary search over node_off), or ISL_GPU_NONE */
uint32_t isl_gpu_to_node(const isl_engine* e, uint32_t gpu);

/* ---- the hot path ------------------------------------------------------ */
/* Replaces the node loop (:190-227) x findDeviceForASlice (:240-262) x
 * getStartIndexFromPreparedState (:303-384) for n pods at once. `in` and `out`
 * are host buffers of n entries; copies are part of the call. */
int  isl_place_batch(isl_engine* e, uint32_t n, const isl_request* in, isl_result* out);
/* A STREAM of batches in one call: batch i has sizes[i] requests, `in`/`out` hold the batches back to back.
 * Semantics are exactly those of calling isl_place_batch once per batch in order; the engine pipelines the
 * batches over inventory segments (DESIGN.md "Segment pipeline").  Sum of sizes <= isl_config.max_batch.
 * With PINNED host buffers (cudaHostAlloc / cudaHostRegister) the batches are copied and pre-passed while the pipeline
 * already runs and finished chunks are written straight into `out`; pageable buffers work without that overlap.
 * Environment: ISL_NO_FEED=1 switches the overlap off (the library does so itself under kernel-serialising tools). */
int  isl_place_stream(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, const isl_request* in, isl_result* out);
int  isl_place_stream_device(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, const void* d_in, void* d_out);
/* Same, requests and results already resident in device memory (CUdeviceptr as void*). */
int  isl_place_batch_device(isl_engine* e, uint32_t n, const void* d_in, void* d_out);
/* isl_place_batch restricted to the canonical GPU range [lo, hi) — findDeviceForASlice looks at ONE node's GPUs (:240-262), the node
 * loop (:190) calls it node after node.  Restriction, placement and restore happen under one engine lock (two reconcile workers
 * cannot interleave, nothing leaks when the call fails); the engine's own partition (isl_set_partition) is left untouched.
 * Inside a restricted range (this call, isl_set_partition, each node pass of ISL_FLAG_ALL_NODES):
 *   - a well-formed FREE naming a GPU outside [lo, hi) is reported ISL_ST_FREED and NOT applied (the rank that owns the GPU applies it;
 *     the element-wise MIN merge of partitioned results relies on every rank reporting the same FREED record); a malformed one is BAD_SPAN;
 *   - an unplaced ALLOC reports the size of the whole inventory's default row (first node, canonical order, whose table has the name),
 *     not that of the first node of the range;
 *   - an empty range (lo == hi) places nothing: ALLOCs NO_CAPACITY, FREEs FREED and not applied, on every policy. */
int  isl_place_batch_range(isl_engine* e, uint32_t lo, uint32_t hi, uint32_t n, const isl_request* in, isl_result* out);
/* All-or-nothing pod groups (the replicas of a deployment, the workers of a job).  `in` / `out` hold n = gang_off[n_gangs] requests and
 * records (host buffers, as isl_place_batch); gang i is in[gang_off[i] .. gang_off[i + 1]), gang_off[0] == 0, no gang is empty.
 *   1. Every FREE of the call is applied first, wherever it is listed (FREED / BAD_SPAN); a FREE never aborts a gang.  NOOP members
 *      report NOOP and do not count.
 *   2. Gangs in array order; inside a gang the ALLOC members are resolved in order by the engine's policy, each one seeing every commit
 *      before it, tentative ones of its own gang included.  A gang of one ALLOC is an ordinary request.
 *   3. A gang whose ALLOC members are all placed commits: the usual PLACED records.
 *   4. Otherwise the first member that cannot be placed gets its usual record (NO_CAPACITY, or BAD_PROFILE for an unknown profile), the
 *      members after it are not tried, and every other ALLOC member of the gang reports ISL_ST_GANG_ABORTED with the unplaced default
 *      record (gpu ISL_GPU_NONE, start 9, the profile's size or 0 for an unknown profile).
 *   5. The occupancy after an aborted gang is exactly what it was before it: later gangs see no trace of it.
 *   6. Every policy, both quirk sets and per-node tables; inside the engine's partition (isl_set_partition).  Stats count committed
 *      placements only.
 * A call whose gangs all have one member equals isl_place_batch on the same requests, records and occupancy.  The gangs are resolved
 * request by request (the best-fit kernel's loop, DESIGN.md 4.6): first-fit gangs do not use the segment pipeline.
 * ISL_EINVAL: malformed offsets, NULL buffers, an engine created with ISL_FLAG_ALL_NODES.  ISL_ERANGE: n > max_batch, or a partition
 * that is empty or holds more than 2^20 GPUs.  ISL_ESTATE: no profiles or inventory, or an open stream. */
int  isl_place_gangs(isl_engine* e, uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out);

/* ---- open streams: the causal feed --------------------------------------- */
/* A reconciler that composes batch b+1 from the results of batch b (a FREE names an allocation an earlier batch placed) cannot hand
 * all batches over up front.  An open stream keeps ONE persistent pipeline kernel resident:
 *   isl_stream_open(e, max_batches)            reserve tables for up to max_batches batches of <= 65 536 requests
 *   isl_stream_submit(e, n, in, out, &ticket)  enqueue one batch: copy + pre-pass on the feed stream; returns at once.  `out` must be
 *                                              mapped pinned host memory (isl_host_alloc / cudaHostAlloc / cudaHostRegister): the
 *                                              running kernel writes the results there
 *   isl_stream_wait(e, ticket)                 returns when that batch's results are in `out`
 *   isl_stream_close(e)                        end of stream: the kernel drains, the occupancy is written back
 * Results are exactly those of isl_place_batch per batch in submission order.  Batches submitted before earlier ones are waited for
 * overlap on the device (segment pipeline).  While a stream is open every other call on the engine returns ISL_ESTATE. */
int  isl_stream_open(isl_engine* e, uint32_t max_batches);
int  isl_stream_submit(isl_engine* e, uint32_t n, const isl_request* in, isl_result* out, uint32_t* ticket);
int  isl_stream_wait(isl_engine* e, uint32_t ticket);
int  isl_stream_close(isl_engine* e);
/* Device-side causal window for isl_place_stream / isl_place_stream_device: batch b is not started before every inventory segment has
 * committed batch b - window (0 = no constraint, the default).  Models a consumer that needs batch b - window's results to compose b. */
int  isl_set_causal_window(isl_engine* e, uint32_t window);
/* Speculative rounds inside the segment pipeline: a batch's decisions are ONE recurrence over the inventory (the reference's
 * first-fit in arrival order, :240-262), so a batch that must be resolved before the next one may start keeps all inventory stages but
 * one idle.  With speculation every stage simulates its segment at once from PREDICTED queue heads, the predictions are corrected
 * round by round and a stage commits only when its entry is certified to be the true one — results are bit-identical, a batch's
 * latency drops from (stages x segment time) to (rounds x segment time).  It pays when few batches may be in flight and costs
 * throughput when many may overlap anyway:
 *   ISL_SPEC_AUTO (default)  single batches and streams with a causal window of 1..3; open streams: when a window of 1..3 is set
 *   ISL_SPEC_OFF / ISL_SPEC_ON  never / whenever the geometry allows it: one sub-segment per inventory stage (<= 132 x 512 = 67 584 GPUs per
 *                            engine; larger inventories keep the plain pipeline), a partitioned inventory only with isl_ipc_connect_spec */
#define ISL_SPEC_AUTO 0u
#define ISL_SPEC_OFF  1u
#define ISL_SPEC_ON   2u
int  isl_set_speculation(isl_engine* e, uint32_t mode);
/* Mapped pinned host memory from the C side (cgo must not hand Go-heap pointers to a running kernel). NULL on failure. */
void* isl_host_alloc(size_t bytes);
void  isl_host_free(void* p);
/* Releases spans (Allocations entries deleted by the daemonset). */
int  isl_free_batch(isl_engine* e, uint32_t n, const isl_span* spans);
/* getStartIndexFromPreparedState's search (:343-383) for n arbitrary occupancy
 * bytes and one profile row, evaluated by the device table: out[i] in {0..7, 9}.  `profile` = name index | table << 8. */
int  isl_eval_starts(isl_engine* e, uint32_t profile, uint32_t n, const uint8_t* occ, uint8_t* out);

/* ---- partitioned inventory (BASELINE config 4; DESIGN.md "Multi-GPU") ---- */
/* Restrict this engine to the canonical GPU range [lo, hi) of the loaded
 * inventory.  The batch is resolved by chaining ranks in range order: rank d
 * starts from the per-profile queue heads rank d-1 ended with.  Every single-engine entry point (batch, stream, open stream,
 * isl_capacity, isl_what_if, isl_free_batch, gangs, the best-fit family) then sees [lo, hi) only, with the FREE and default-size rules
 * of isl_place_batch_range; isl_free_batch skips spans outside the partition. */
int  isl_set_partition(isl_engine* e, uint32_t lo, uint32_t hi);
/* d_heads_in / d_heads_out: ISL_MAX_PROFILES uint32 each in device memory
 * (NULL d_heads_in = first rank).  Results of requests this rank did not place
 * keep status NO_CAPACITY / gpu NONE so that an elementwise MIN over ranks of the
 * 8-byte records (as little-endian uint64) yields the global answer. */
int  isl_place_batch_partitioned(isl_engine* e, uint32_t n, const void* d_in, void* d_out,
                                 const void* d_heads_in, void* d_heads_out);
/* Stream variant for a partitioned inventory, one engine (process, GPU) per rank, ranks ordered by GPU range.
 * The queue-head token of every chunk crosses from the last segment of rank d to the first segment of rank d+1
 * through rank d+1's inbox, mapped into rank d with CUDA IPC (a peer store over NVLink inside the running kernel):
 *   1. every rank:  isl_ipc_inbox_handle(e, h)             -> 64-byte handle, exchanged by the caller (e.g. all_gather)
 *   2. every rank:  isl_ipc_connect(e, next rank's handle or NULL for the last rank, has_prev)
 *   3. every rank:  isl_place_stream_partitioned(..., stream_id) with the same batches and the same non-zero,
 *      never repeated stream_id (it tags what crosses the ranks; the speculative rounds use its low 24 bits); only enqueues.  Results: element-wise MIN over ranks as for the batch variant. */
int  isl_ipc_inbox_handle(isl_engine* e, void* handle64);
int  isl_ipc_connect(isl_engine* e, const void* next_handle64, int has_prev);
/* Same wiring for two engines of ONE process (same device or peer-enabled devices): no IPC handle needed. */
int  isl_connect_local(isl_engine* e, isl_engine* next, int has_prev);
int  isl_place_stream_partitioned(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, const void* d_in, void* d_out,
                                  uint32_t stream_id);
/* Device address of the occupancy bytes owned by this engine (for the NCCL all-gather). */
void* isl_device_occupancy(isl_engine* e);
/* Results gathered on the owner rank (the controller's rank, rank 0) WITHOUT a collective: every other rank maps the owner's result
 * array and its commit threads store each PLACED record there as well (peer store over NVLink inside the running kernel).  The owner's
 * pre-pass has written the defaults of a batch before its token leaves rank 0, so a later rank's record always lands on top of them.
 *   owner:  isl_ipc_results_handle(e, h) -> 64-byte handle; place with d_out = isl_device_results(e)
 *   others: isl_ipc_connect_owner(e, h) (NULL disconnects); same-process engines: isl_connect_owner_local
 * A collective or barrier that every rank enqueues behind its kernel (e.g. the occupancy all-gather) tells the owner that all records
 * have arrived. */
void* isl_device_results(isl_engine* e);
int  isl_ipc_results_handle(isl_engine* e, void* handle64);
int  isl_ipc_connect_owner(isl_engine* e, const void* owner_handle64);
int  isl_connect_owner_local(isl_engine* e, isl_engine* owner);
/* Speculative rounds (isl_set_speculation) over a partitioned inventory: the stages of all ranks form one sequence and exchange their
 * per-round records through peer memory, so every rank maps every other rank's record memory.
 *   every rank:  isl_ipc_spec_handle(e, h)                  -> 64-byte handle of its record memory (allocates it)
 *   every rank:  isl_ipc_connect_spec(e, world, rank, handles [world x 64 bytes], bounds [world + 1])
 * bounds[r] .. bounds[r + 1] is the canonical GPU range of rank r (what isl_set_partition got).  Without it a partitioned stream keeps
 * the token ring.  world = 0 disconnects.  isl_connect_spec_local: same-process engines. */
int  isl_ipc_spec_handle(isl_engine* e, void* handle64);
int  isl_ipc_connect_spec(isl_engine* e, uint32_t world, uint32_t rank, const void* handles, const uint32_t* bounds);
int  isl_connect_spec_local(isl_engine* e, uint32_t world, uint32_t rank, isl_engine* const* engines, const uint32_t* bounds);
/* Number of ranks of the partitioned run.  With it set (and the owner's results mapped on every other rank) isl_set_causal_window also
 * applies to isl_place_stream_partitioned: the rank that finishes a chunk adds 1 to a per-chunk counter behind the owner's result
 * array (peer atomic), and the owner starts chunk c only when all `world` ranks are through with chunk c - window.  All ranks must be
 * created with the same isl_config.max_batch. */
int  isl_set_ring_world(isl_engine* e, uint32_t world);

/* ---- diagnostics ------------------------------------------------------- */
int         isl_get_stats(isl_engine* e, isl_stats* out);
/* ISL_FLAG_TRACE: uint64 [chunk][segment][12] of the last stream call = globaltimer ns of local sweep done, token arrived,
 * token published, commit done, decision loop start, decision loop end; decisions of the cell; jumps | GPUs visited << 32;
 * ns of heads computed, queue windows staged; two spare words.
 * out may be NULL to query the dimensions. */
int         isl_read_trace(isl_engine* e, uint64_t* out, uint32_t max_words, uint32_t* n_chunks, uint32_t* n_seg);
int         isl_reset_stats(isl_engine* e);
const char* isl_strerror(int code);
const char* isl_last_cuda_error(const isl_engine* e);
uint32_t    isl_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* ISLPLACE_H */
