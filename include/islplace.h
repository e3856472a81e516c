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
/* Node scoring: the kube-scheduler's NodeResourcesFit strategies, which never apply to gated MIG pods, over the NODES of the range.
 * MOST_ALLOCATED packs pods onto the fullest nodes (so that the cluster autoscaler can drain the emptiest), LEAST_ALLOCATED (the
 * scheduler's default) spreads them.  Batch semantics are unchanged: FREEs first, then the ALLOCs in array order, each seeing every
 * earlier commit.  For one ALLOC of profile name p:
 *   1. Candidate nodes: a node with at least one GPU inside the call's range (the partition, isl_place_batch_range) whose occupancy byte
 *      has a start for p in the start search of its node's table (under the engine's quirk set).  GPUs outside the range do not exist for
 *      the call, also on a node the range cuts.  An empty node is never a candidate.
 *   2. Capacity and usage in MIG memory slices: width(t) = the largest start + size over the rows of table t (8 for the A100 / H100 /
 *      B200 tables, 4 for A30); cap(N) = width(t_N) x the node's GPUs in range; busy(N) = the sum over those GPUs of
 *      popcount(occ & ((1 << width) - 1)); req = the size of p's row in the node's table.
 *   3. Score, NodeResourcesFit's integer formulas with one resource of weight 1 and MaxNodeScore 100:
 *      MOST_ALLOCATED floor(100 x (busy + req) / cap), LEAST_ALLOCATED floor(100 x (cap - busy - req) / cap).  On a candidate
 *      busy + req <= cap, and a table without rows (width 0) has no candidate.
 *   4. The highest score wins, ties to the lowest canonical node index (the scheduler picks at random among ties; the engine is
 *      deterministic).  Inside the node the reference's own search decides (findDeviceForASlice on one node, :240-262): the first GPU
 *      in canonical order, within the range, whose byte admits p, and its first legal start in row order.
 *   5. The usual records: PLACED (gpu, start, size); NO_CAPACITY with the default size when no node is a candidate; BAD_PROFILE;
 *      FREED / BAD_SPAN / NOOP.  Stats count as for the best-fit family.
 *   6. Accepted by isl_place_batch, _range, _device, isl_place_stream, _device (one batch after the other), isl_what_if, isl_capacity,
 *      isl_free_batch, isl_eval_starts, isl_set_partition, per-node tables and isl_preempt (whose scan order is ascending canonical).
 *   7. isl_create: ISL_EINVAL with ISL_FLAG_ALL_NODES (a pod placed on every node has no node to choose), ISL_ERANGE for
 *      max_gpus > 2^20.  isl_load_inventory: ISL_ERANGE for more than 2^20 nodes, empty nodes included (the nodes, not the GPUs,
 *      are the leaves of the score trees); the previous inventory stays loaded.  ISL_EINVAL from isl_place_batch_partitioned,
 *      isl_place_stream_partitioned, isl_stream_open, and isl_place_gangs without ISL_FLAG_GANG_NODE_SCORE (N1-N8).
 * On an inventory of one node both give exactly ISL_POLICY_FIRST_FIT's records and occupancy. */
#define ISL_POLICY_MOST_ALLOCATED  4u
#define ISL_POLICY_LEAST_ALLOCATED 5u

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
#define ISL_ST_GANG_TRIMMED 7u  /* not placed: its elastic gang committed its leading members without it (ISL_FLAG_GANG_MIN_MEMBERS, M3) */

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
                                       a compatibility mode for parity studies, not a fast path.  isl_place_batch_range and isl_what_if
                                       follow it; the stream calls and isl_place_batch_device place each pod once, isl_place_gangs is EINVAL */
#define ISL_FLAG_GANG_ONE_NODE 64u  /* isl_place_gangs puts every member of a gang on ONE node (see isl_place_gangs); every other call is unchanged */
#define ISL_FLAG_GANG_DISTINCT_NODES 128u  /* isl_place_gangs puts every member of a gang on a DIFFERENT node (see isl_place_gangs); every
                                              other call is unchanged */
#define ISL_FLAG_GANG_FEW_NODES 256u  /* isl_place_gangs puts a gang on ONE node when one takes it, else on as FEW nodes as it greedily can
                                         (see isl_place_gangs); every other call is unchanged */
#define ISL_FLAG_GANG_LOCALITY 512u  /* isl_place_gangs takes each gang's node locality from its ALLOC members' `start` byte, one of the
                                        ISL_GANG_* values below (see isl_place_gangs); every other call is unchanged */
#define ISL_FLAG_GANG_MIN_MEMBERS 1024u  /* elastic gangs: isl_place_gangs commits a gang's leading members once they reach the minimum its
                                            ALLOC members name in their `size` byte (see isl_place_gangs, M1-M7); every other call is unchanged */
#define ISL_FLAG_GANG_PREEMPT 2048u  /* isl_preempt reads gangs from its requests (runs of equal `handle`) and picks the victims a whole gang
                                        needs, or evicts nothing for it (see isl_preempt, P1-P8); every other call is unchanged */
#define ISL_FLAG_GANG_NODE_SCORE 4096u  /* on a node-scoring engine isl_place_gangs places gangs by MostAllocated or LeastAllocated (see
                                           isl_place_gangs, N1-N8); every other call is unchanged */
#define ISL_FLAG_GANG_BALANCED 8192u  /* with ISL_FLAG_GANG_LOCALITY: a locality byte of 4..255 spreads a gang's members over the nodes
                                         within a maxSkew of byte - 3 (see isl_place_gangs, B1-B8); every other call is unchanged */
#define ISL_FLAG_GANG_NODE_SCORE_ALL 16384u  /* with ISL_FLAG_GANG_NODE_SCORE: few-node, elastic and balanced gangs are node-scored too
                                                (see isl_place_gangs, C1-C8); every other call is unchanged */
/* Node locality of one gang on an ISL_FLAG_GANG_LOCALITY engine (isl_request.start of its ALLOC members, rules L1-L6) */
#define ISL_GANG_ANY_NODES      0u  /* rules 2-4: members anywhere, as on an engine without a gang flag */
#define ISL_GANG_ONE_NODE       1u  /* G2-G3: every member on one node */
#define ISL_GANG_FEW_NODES      2u  /* F2-F3: one node when one takes the gang, else as few nodes as it greedily can */
#define ISL_GANG_DISTINCT_NODES 3u  /* S2-S4: every member on a different node */
#define ISL_GANG_BALANCED_NODES(max_skew) (3u + (max_skew))  /* B1-B8, ISL_FLAG_GANG_BALANCED: max_skew 1..252 */

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
 * per-(profile, occupancy byte) first-start table on the device.  Loading tables (this call or isl_load_profile_tables) resets every
 * node to table 0: call isl_set_node_tables again after it.  The inventory, the partition and a snapshot are kept. */
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
 * occ has node_off[n_nodes] bytes.  This is also "resume": the CR is the checkpoint.
 * It resets the partition to [0, G), every node to table 0 (isl_set_node_tables) and drops a snapshot (isl_snapshot_occupancy).
 * ISL_ERANGE: node_off[n_nodes] > max_gpus, or more than 2^20 nodes (empty ones included) on a node-scoring engine; a refused
 * call leaves the previous inventory, partition and snapshot in place. */
int  isl_load_inventory(isl_engine* e, uint32_t n_nodes, const uint32_t* node_off, const uint8_t* occ);
int  isl_read_occupancy(isl_engine* e, uint8_t* out /* G bytes */);
/* Incremental sync: overwrite the occupancy bytes of canonical GPUs [first_gpu, first_gpu + n) — what the shim does
 * when ONE Instaslice object changed (an Allocations / Prepared entry appeared or disappeared) instead of re-listing
 * every node (the reference deep-copies the whole list on every reconcile, :85). */
int  isl_write_occupancy(isl_engine* e, uint32_t first_gpu, uint32_t n, const uint8_t* occ);
/* What-if queries (defragmentation planning, SURVEY 8f-4): isl_snapshot_occupancy keeps a device-side copy of the whole
 * occupancy, any number of isl_place_* / isl_free_batch calls then run against the live state, isl_restore_occupancy puts the
 * snapshot back (a 1-byte-per-GPU device copy, no host round trip).  ISL_ESTATE if there is no inventory / no snapshot.
 * A snapshot is the whole occupancy and outlives placement calls, open streams, isl_free_batch, isl_write_occupancy, isl_set_partition
 * and table reloads; isl_load_inventory and isl_what_if drop it, and it can be restored any number of times. */
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
 *   6. Every policy except node scoring (ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED; see ISL_FLAG_GANG_NODE_SCORE, N1-N8), both
 *      quirk sets and per-node tables; inside the engine's partition (isl_set_partition).  Stats count committed placements only.
 * A call whose gangs all have one member equals isl_place_batch on the same requests, records and occupancy.  The gangs are resolved
 * request by request (the best-fit kernel's loop, DESIGN.md 4.6): first-fit gangs do not use the segment pipeline.
 * ISL_EINVAL: malformed offsets, NULL buffers, an engine created with ISL_FLAG_ALL_NODES, or with a node-scoring policy but without
 * ISL_FLAG_GANG_NODE_SCORE.  ISL_ERANGE: n > max_batch, or a partition
 * that is empty or holds more than 2^20 GPUs.  ISL_ESTATE: no profiles or inventory, or an open stream.
 *
 * One-node gangs (ISL_FLAG_GANG_ONE_NODE): pods that talk to each other (a job's workers, a pipeline-parallel deployment) exchange data
 * through host shared memory on one node and through the network across nodes; MIG instances have no peer-to-peer path.  On an engine
 * created with the flag:
 *   G1. Rules 1, 2 (FREEs first, NOOPs ignored, gangs in array order), 3 and 5 hold unchanged; rule 6 with the refusals of G5.
 *   G2. A gang commits on the FIRST node, in the engine's scan order (ascending canonical; descending under ISL_POLICY_RIGHT_TO_LEFT), on
 *       which all of its ALLOC members fit.  Inside that node the members are resolved in order by the engine's policy restricted to the
 *       node's GPUs inside the partition: first-fit takes the first admitting GPU, right-to-left the last, best-fit and min-frag the
 *       minimum of their score with ties to scan order.  A node the partition cuts offers only its GPUs inside the partition.
 *   G3. Failure record (instead of rule 4): let D be the largest number of leading ALLOC members that any node can place on its own.  If
 *       no node takes the whole gang, the ALLOC member at position D (counting ALLOC members from 0) gets its usual record (NO_CAPACITY,
 *       or BAD_PROFILE for an unknown profile) and every other ALLOC member reports ISL_ST_GANG_ABORTED with the unplaced default
 *       record.  On an inventory of one node this is rule 4.
 *   G4. Consequences: on a one-node inventory, or a partition inside one node, a flagged call equals the unflagged one (records and
 *       occupancy, every policy).  With gangs of one, a flagged ISL_POLICY_FIRST_FIT or _RIGHT_TO_LEFT engine equals isl_place_batch.
 *   G5. isl_create: ISL_EINVAL for the flag with ISL_FLAG_ALL_NODES or a node-scoring policy.  isl_place_gangs keeps every code above,
 *       the 2^20-GPU partition cap included.  Every other entry point returns exactly what it returns on an unflagged engine.
 *   G6. The flag applies to every gang of the engine.  To choose node locality gang by gang, use ISL_FLAG_GANG_LOCALITY (L1-L6).
 *
 * Distinct-node gangs (ISL_FLAG_GANG_DISTINCT_NODES): the replicas of a deployment on different nodes, so that one node or one GPU
 * failing does not take down every replica (the kube-scheduler's required podAntiAffinity on kubernetes.io/hostname, which never applies
 * to gated MIG pods).  On an engine created with the flag:
 *   S1. Rules 1, 2 (FREEs first, NOOPs ignored, gangs in array order), 3 and 5 hold unchanged; rule 6 with the refusals of S6.
 *   S2. Inside a gang the ALLOC members are resolved in order, each by the engine's policy restricted to the GPUs of the partition whose
 *       node holds no earlier member of the SAME gang: first-fit takes the first admitting GPU in ascending canonical order,
 *       right-to-left the last, best-fit and min-frag the minimum of their score with ties to scan order; the start inside the GPU is
 *       the start search's.  A node the partition cuts counts as one node and offers only its GPUs inside the partition.  Nodes used by
 *       earlier committed gangs are not excluded: the anti-affinity holds within one gang.
 *   S3. Failure is rule 4 unchanged: the first member with no admitting GPU on an unused node gets its usual record (NO_CAPACITY, or
 *       BAD_PROFILE for an unknown profile), the members after it are not tried, and every other ALLOC member reports
 *       ISL_ST_GANG_ABORTED with the unplaced default record.  NO_CAPACITY may be reported while a node the gang already uses has room.
 *   S4. The choice is greedy, member by member, not a matching (the kube-scheduler placing pods with required anti-affinity one at a
 *       time): a gang can abort although some assignment to distinct nodes exists.  Node A admits 1g and 4g, node B only 1g: under
 *       first-fit [1g, 4g] aborts (1g takes A) while [4g, 1g] places.  List the larger members of a gang first.
 *   S5. Consequences: (a) with gangs of one, a flagged call equals isl_place_batch (records and occupancy, every policy); (b) the PLACED
 *       members of a committed gang sit on pairwise distinct nodes (isl_gpu_to_node); (c) a gang with more ALLOC members than the
 *       partition has non-empty nodes always aborts, so on a one-node inventory every gang of two or more ALLOC members aborts (when
 *       member 0 places, member 1 reports NO_CAPACITY); (d) on an inventory of one-GPU nodes under ISL_QUIRKS_FIXED with gangs whose
 *       profiles all take a whole GPU (size 8), a flagged call equals the unflagged one on every policy.
 *   S6. isl_create: ISL_EINVAL for the flag with ISL_FLAG_GANG_ONE_NODE (they contradict each other), ISL_FLAG_ALL_NODES or a
 *       node-scoring policy.  isl_place_gangs keeps every code above, the 2^20-GPU partition cap included.  Every other entry point
 *       returns exactly what it returns on an unflagged engine.  The flag applies to every gang of the engine, as G6 says.
 *
 * Few-node gangs (ISL_FLAG_GANG_FEW_NODES): a job's workers that should share a node but must still run when no single node has room for
 * them (Kueue's preferred topology on kubernetes.io/hostname, which never applies to gated MIG pods).  On an engine created with the flag:
 *   F1. Rules 1, 2 (FREEs first, NOOPs ignored, gangs in array order), 3 and 5 hold unchanged; rule 6 with the refusals of F6.
 *   F2. Rounds.  Let m_0 .. m_{k-1} be the gang's ALLOC members and i = 0.  In each round d(node) is how many of the leading members
 *       m_i, m_{i+1}, .. the node places, resolved in order by the engine's policy restricted to that node's GPUs inside the partition,
 *       exactly as in G2, on the occupancy left by committed gangs and by this gang's earlier rounds (a node the partition cuts offers
 *       only its GPUs inside the partition).  The node with the largest d takes m_i .. m_{i+d-1}, ties to the first node in scan order
 *       (ascending canonical; descending under ISL_POLICY_RIGHT_TO_LEFT); then i += d.  The gang commits when i = k.  A node that takes
 *       every remaining member has the largest possible d, so when some node takes them all, the first such node wins, as in G2.
 *   F3. Failure: when the largest d of a round is 0, member m_i gets its usual record (NO_CAPACITY, or BAD_PROFILE for an unknown
 *       profile) and every other ALLOC member reports ISL_ST_GANG_ABORTED with the unplaced default record.  The occupancy is what it was
 *       before the gang (rule 5), the slices of its earlier rounds included.
 *   F4. Consequences: (a) a gang that some single node takes whole gets exactly the records and occupancy of a GANG_ONE_NODE engine (round
 *       1 is G2); (b) a gang that fails here fails on a GANG_ONE_NODE engine in the same state; (c) on a one-node inventory, or a partition
 *       inside one node, a flagged call equals the unflagged one (records and occupancy, every policy): the second round on the same node
 *       has d = 0 at the member that did not fit, which is rule 4; (d) with gangs of one, a flagged call equals a GANG_ONE_NODE call, and
 *       under ISL_POLICY_FIRST_FIT and _RIGHT_TO_LEFT isl_place_batch; (e) two consecutive rounds never use the same node (the member that
 *       ended round r does not fit on its node, so that node has d = 0 next), so the maximal runs of a committed gang's ALLOC members on
 *       one node (isl_gpu_to_node) are exactly its rounds.  A node may come back in a later, non-adjacent round when a smaller member fits
 *       where an earlier one did not: A100-40GB tables, reference-exact quirks, one-GPU nodes with bytes 0x01 and 0xF0, first-fit gang
 *       [1g.5gb, 3g.20gb, 1g.5gb] commits on nodes 0, 1, 0 where a GANG_ONE_NODE engine aborts it.
 *   F5. The choice is greedy, round by round (Kueue's largest domain first), not a minimum cover, and a tie goes to scan order even when
 *       an earlier round already uses one of the tied nodes: the gang may use more nodes than it needs.  A100-40GB tables, reference-exact
 *       quirks, first-fit, one-GPU nodes with bytes 0xF0, 0x0F and 0x80, gang [4g.20gb, 2g.10gb, 3g.20gb, 1g.5gb]: node 2 takes the
 *       first two members (d = [1, 0, 2]), node 0 the 3g.20gb, and node 1 the last 1g.5gb (a tie with node 2): three nodes, where
 *       node 2 could have taken the last member too.
 *   F6. isl_create: ISL_EINVAL for the flag with ISL_FLAG_GANG_ONE_NODE, ISL_FLAG_GANG_DISTINCT_NODES, ISL_FLAG_ALL_NODES or a
 *       node-scoring policy.  isl_place_gangs keeps every code above, the 2^20-GPU partition cap included.  Every other entry point
 *       returns exactly what it returns on an unflagged engine.  The flag applies to every gang of the engine, as G6 says.
 *
 * Node locality per gang (ISL_FLAG_GANG_LOCALITY): one burst of pending pods that mixes a job needing one node, replicas that must sit on
 * distinct nodes, a job that prefers few nodes and pods that go anywhere (Kueue's per-workload podset-required-topology and
 * podset-preferred-topology), placed by one call on one occupancy.  On an engine created with the flag:
 *   L1. An ALLOC member's `start` byte names its gang's locality: ISL_GANG_ANY_NODES (0), _ONE_NODE (1), _FEW_NODES (2) or
 *       _DISTINCT_NODES (3).  A FREE's `start` stays its span; a NOOP's is ignored.  A gang with no ALLOC member has no locality.
 *   L2. Rules 1, 3 and 5 hold unchanged.  Rule 2's order holds across localities: gangs go in array order, and each gang sees every
 *       commit of every earlier gang, whatever that gang's locality.  Each gang is placed by the rules of its locality, on the
 *       occupancy that the call's FREEs and the earlier gangs left: 0 by rules 2-4 (as on an engine without a gang flag), 1 by G2-G3,
 *       2 by F2-F3, 3 by S2-S4.
 *   L3. Consequences: (a) a call whose ALLOC members all carry locality k equals isl_place_gangs on an engine created with k's flag (no
 *       gang flag for 0), with the same policy, quirks, node tables and partition: records, occupancy and stats.placed; (b) a call equals
 *       its gangs run one at a time, each alone on the engine flagged for its locality, after the call's FREEs, with the occupancy handed
 *       on from each gang to the next; (c) with every byte 0, under ISL_POLICY_FIRST_FIT or _RIGHT_TO_LEFT, gangs of one equal
 *       isl_place_batch.
 *   L4. ISL_EINVAL, and nothing changes, when an ALLOC's byte is greater than 3 or two ALLOC members of one gang name different
 *       localities.  These checks run with the other argument checks, before the engine state is looked at.
 *   L5. isl_create: ISL_EINVAL for the flag with ISL_FLAG_GANG_ONE_NODE, _DISTINCT_NODES, _FEW_NODES, ISL_FLAG_ALL_NODES or a
 *       node-scoring policy.  isl_place_gangs keeps every code above, the 2^20-GPU partition cap included.  Every other entry point
 *       returns exactly what it returns on an unflagged engine.
 *   L6. Locality matters even for a gang of one: under best-fit a one-node gang of one takes the best GPU of the FIRST node in scan order
 *       that admits it, not the best GPU of the whole partition. */
/*
 * Elastic gangs (ISL_FLAG_GANG_MIN_MEMBERS): a group of k pods that may run as soon as m <= k of them can (the coscheduling plugin's
 * PodGroup minMember, Volcano's minAvailable, Kueue's partial admission; elastic training and inference replicas).  On an engine created
 * with the flag, alone or with one of the four gang flags above:
 *   M1. An ALLOC member's `size` byte names its gang's minimum m (0..255); every ALLOC member of one gang carries the same byte.  With k
 *       the gang's ALLOC members, the effective minimum is m' = k when m = 0 or m >= k, else m' = m, so m' >= 1.  A FREE's `size` stays
 *       its span and a NOOP's is ignored.  Under ISL_FLAG_GANG_LOCALITY the `start` byte still names the locality (L1).
 *   M2. The gang is placed by the rules of its locality exactly as without the flag: rules 2-4 with no gang flag, G2-G3 one node, F2-F3
 *       few nodes, S2-S4 distinct nodes, per gang under ISL_FLAG_GANG_LOCALITY.  A gang those rules commit is unchanged.
 *   M3. Trimming.  When those rules fail at ALLOC member f (counted from 0; the member that keeps its usual record: rule 4, G3's D, F3's
 *       m_i, S3) and f >= m', the gang commits its first f ALLOC members where the run put them (rules 2-4 and S: member by member; G:
 *       on the first node in scan order that reaches depth D; F: the rounds so far), with PLACED records.  Member f keeps its usual
 *       record (NO_CAPACITY or BAD_PROFILE); every ALLOC member after it reports ISL_ST_GANG_TRIMMED with the unplaced default record
 *       (gpu ISL_GPU_NONE, start 9, the profile's size or 0 for an unknown profile).  stats.placed counts the f members.
 *   M4. When f < m' the gang aborts exactly as without the flag (rule 4 / G3 / F3 / S3 and rule 5): f = 0 always aborts.
 *   M5. Consequences: (a) with every byte 0, or every byte >= its gang's k, a flagged call equals the call on the engine without the
 *       flag (records, occupancy, stats.placed) for every gang flag and none; (b) a gang trimmed at f gets exactly the records and
 *       occupancy that the gang cut to its first f ALLOC members gets without the flag, and that cut gang commits; (c) under
 *       ISL_FLAG_GANG_LOCALITY a call equals its gangs run one at a time, each on the engine flagged for its locality | MIN (L3 b);
 *       (d) gangs of one ALLOC member are unaffected.
 *   M6. isl_create: ISL_EINVAL for the flag with ISL_FLAG_ALL_NODES or a node-scoring policy (the four gang flags keep their own
 *       refusals, so at most one of them comes with it).  isl_place_gangs: ISL_EINVAL, and nothing changes, when two ALLOC members of
 *       one gang carry different bytes, checked with L4 before the engine state is looked at; every other code is unchanged, the
 *       2^20-GPU partition cap included.  Every other entry point returns what it returns on an unflagged engine.
 *   M7. The committed members are always a LEADING run, never the best subset: under first-fit a gang [4g, 1g, 1g] with m = 2 aborts
 *       when the 4g fits nowhere, although both 1g would fit.  List the members the job needs first; for replicas of one profile the
 *       leading run is as many members as the locality places.
 *
 * Node-scored gangs (ISL_FLAG_GANG_NODE_SCORE): a cluster that packs its pods with MostAllocated (so that the autoscaler can drain the
 * emptiest nodes) or spreads them with LeastAllocated places its jobs and replicas as gangs on the same engine, the same inventory and
 * the same lock as its single pods, and a one-node gang goes to the fullest (emptiest) node that takes it, not the first.  On an engine
 * created with the flag:
 *   N1. isl_create: ISL_EINVAL for the flag without ISL_POLICY_MOST_ALLOCATED or _LEAST_ALLOCATED, or with ISL_FLAG_GANG_FEW_NODES or
 *       ISL_FLAG_GANG_MIN_MEMBERS, unless ISL_FLAG_GANG_NODE_SCORE_ALL is set as well (C1; ISL_FLAG_ALL_NODES is refused by node
 *       scoring already).  It may come with at most one of
 *       ISL_FLAG_GANG_ONE_NODE, _DISTINCT_NODES and _LOCALITY (their mutual refusals are unchanged; only their refusal of node scoring is
 *       lifted, and only with this bit), and with ISL_FLAG_GANG_PREEMPT (N7).  max_gpus > 2^20 and more than 2^20 nodes keep node
 *       scoring's ISL_ERANGE.
 *   N2. Rules 1, 2, 3 and 5 hold.  A gang's locality is the engine's flag, under ISL_FLAG_GANG_LOCALITY its ALLOC members' `start` byte
 *       (L1), with neither any node.
 *   N3. Any node: the ALLOC members in order, each placed by node-scoring rules 1-5 over the partition with req = its own row size, each
 *       seeing every earlier commit, the gang's tentative members included (their slices count in busy).  Failure is rule 4.
 *   N4. Distinct nodes: each member as in N3, restricted to the nodes that hold no earlier member of the same gang (a node the partition
 *       cuts counts as one node, as in S2).  Failure is S3; the choice is greedy, member by member (S4).
 *   N5. One node: node N can take the gang when its ALLOC members, resolved in order by the reference's search restricted to N's GPUs
 *       inside the partition, all place.  Among those nodes the gang goes to the highest score for req = R(N), the sum of the members'
 *       row sizes in N's table (the gang scored as one pod, as P3 does): MostAllocated floor(100 (busy + R) / cap), LeastAllocated
 *       floor(100 (cap - busy - R) / cap); ties to the lowest canonical node index.  With no such node the failure record is G3 (same D).
 *   N6. Both quirk sets, per-node tables (each node's score normalised by its own width), inside isl_set_partition; stats.placed counts
 *       committed members only.  isl_place_gangs keeps every code above, the 2^20-GPU partition cap included.  Under
 *       ISL_FLAG_GANG_LOCALITY a locality byte of 2 (few nodes) is ISL_EINVAL, checked with L4 before the engine state is looked at;
 *       nothing changes.  ISL_FLAG_GANG_NODE_SCORE_ALL lifts this (C2).
 *   N7. Every other entry point returns exactly what it returns on the same engine without the bit: isl_place_batch and every other
 *       k_nodefit caller, isl_what_if, isl_capacity, isl_preempt.  With ISL_FLAG_GANG_PREEMPT, isl_preempt keeps P1-P8, whose scan
 *       order is ascending canonical under node scoring (rule 5), so it returns what a FIRST_FIT engine with the same flags minus this
 *       one returns.
 *   N8. Consequences: (a) with gangs of one ALLOC member, a call of any locality (0, 1 or 3) equals isl_place_batch on the same engine:
 *       records, occupancy and stats.placed; (b) under any-node locality a call equals its gangs run one at a time: a committed gang
 *       equals isl_place_batch of its ALLOC members on the occupancy before it, an aborted gang changes nothing; (c) on a one-node
 *       inventory, or a partition inside one node, a call equals isl_place_gangs on a FIRST_FIT engine with the same locality flags,
 *       records and occupancy (on one node node scoring is first-fit); (d) a committed one-node gang's members share a node, a committed
 *       distinct-node gang's members sit on pairwise distinct nodes (isl_gpu_to_node).
 *   Example, H100-80GB rows (width 8), either quirk set: three one-GPU nodes with bytes 0x00, 0x3F and 0x0F, gang [1g.10gb, 1g.10gb].
 *       one node        MOST: GPU 2 at starts 4, 5 (node 1 is fullest but start 7 is not legal, so it takes one member; R = 2 scores
 *                       node 0 25 and node 2 75).  LEAST: GPU 0 at starts 0, 1 (75 against 25).  First-fit would take node 0.
 *       any node        MOST: GPU 1 start 6 (87 against 12 and 62), then GPU 2 start 4 (node 1, now 0x7F, admits no 1g.10gb).
 *                       LEAST: GPU 0 starts 0 then 1.
 *       distinct nodes  MOST: as any node.  LEAST: GPU 0 start 0, then GPU 2 start 4 (node 0 is used; 37 against node 1's 12).
 *
 * Balanced gangs (ISL_FLAG_GANG_BALANCED): the replicas of a deployment spread over the nodes for availability, but more of them than
 * there are nodes (Kubernetes' topologySpreadConstraints with maxSkew k on kubernetes.io/hostname, which never applies to gated MIG
 * pods).  Any-node gangs pack them onto the first GPU with room, and distinct-node gangs abort once every node holds one.  On an engine
 * created with the flag:
 *   B1. The flag is valid only with ISL_FLAG_GANG_LOCALITY.  An ALLOC member's `start` byte b of 4..255 makes its gang a balanced gang
 *       with maxSkew k = b - 3 (1..252; ISL_GANG_BALANCED_NODES(k)).  Bytes 0..3 keep L1's meaning, and two ALLOC members of one gang
 *       with different bytes are ISL_EINVAL (L4).  Without the flag L4 is unchanged: a byte above 3 is ISL_EINVAL.
 *   B2. Rules 1, 3 and 5 hold, and so does L2's order across localities.  A balanced gang's ALLOC members are resolved in order, each
 *       seeing the gang's earlier members as tentative slices (rules 2-4); two members may share a GPU.  For a member of profile p,
 *       cnt(N) is the number of earlier ALLOC members of the same gang placed on node N, A is the set of the partition's nodes with a GPU
 *       inside the partition whose current byte admits p under the start search of the node's table, and mu = the least cnt over A.  The
 *       candidates are the admitting GPUs of the nodes N of A with cnt(N) <= mu + k - 1, and the engine's policy picks among them:
 *       first-fit the first in ascending canonical order, right-to-left the last, best-fit and min-frag the minimum of their score with
 *       ties to scan order.  The start is the start search's.  A node the partition cuts counts as one node and offers only its GPUs
 *       inside the partition, as in S2.
 *   B3. Failure is rule 4: the first member with no admitting GPU anywhere in the partition keeps its NO_CAPACITY or BAD_PROFILE record,
 *       every other ALLOC member reports ISL_ST_GANG_ABORTED, and the occupancy is what it was before the gang.  The skew never causes a
 *       failure: a node at mu always qualifies.
 *   B4. Consequences: (a) a gang that commits whole with byte 3 gets the same records with byte 4 (k = 1): while an unused admitting node
 *       exists, mu = 0 and the candidates are S2's; (b) byte 3 + k with k >= the gang's ALLOC members equals byte 0; (c) on a one-node
 *       inventory, or a partition inside one node, every balanced byte equals byte 0; (d) gangs of one equal byte 0, and under FIRST_FIT
 *       and RIGHT_TO_LEFT isl_place_batch; (e) L3 (b) extends: a call equals its gangs run one at a time; (f) with k = 1, on an inventory
 *       where every node admits every member until the gang ends, the final per-node counts differ by at most 1.
 *   B5. Elastic gangs: with ISL_FLAG_GANG_MIN_MEMBERS, M3 applies member by member, as for S: with f the rank of the first member with
 *       no admitting GPU, the gang commits its leading f members when f >= m'.
 *   B6. isl_create: ISL_EINVAL for the flag without ISL_FLAG_GANG_LOCALITY, with a node-scoring policy (hence with
 *       ISL_FLAG_GANG_NODE_SCORE) unless ISL_FLAG_GANG_NODE_SCORE_ALL is set (C1), or with ISL_FLAG_ALL_NODES.  ISL_FLAG_GANG_PREEMPT may come with it; isl_preempt keeps P1, which refuses
 *       bytes above 3, so no balanced gang is preempted for.  isl_place_gangs keeps every other code, the 2^20-GPU partition cap
 *       included.  Every other entry point returns exactly what it returns without the flag.
 *   B7. The choice is greedy, member by member (as S4 and F5): list the larger members first.
 *   B8. Deliberate difference from PodTopologySpread: mu is taken over the nodes that still admit the member, not over every node (a
 *       full node would otherwise hold the minimum at its count, and DoNotSchedule would refuse every later member elsewhere); and the
 *       counts are within the gang: replicas placed by earlier calls are not counted, as S2 ignores them.
 *   Example, H100-80GB rows, either quirk set, two one-GPU nodes with bytes 0x00 and 0x00, a gang of four 1g.10gb, records (gpu, start):
 *       byte 0        first-fit (0,0) (0,1) (0,2) (0,3)
 *       byte 3        member 2 NO_CAPACITY, members 0, 1 and 3 GANG_ABORTED (they had reached (0,0) and (1,0))
 *       byte 4 (k 1)  first-fit (0,0) (1,0) (0,1) (1,1); right-to-left (1,0) (0,0) (1,1) (0,1)
 *       byte 5 (k 2)  first-fit (0,0) (0,1) (1,0) (0,2)
 *       byte 7 (k 4)  equals byte 0
 *   B8's case: three one-GPU nodes with bytes 0x00, 0x7F and 0x00, a gang of three 1g.10gb, byte 4, first-fit: (0,0) (2,0) (0,1).  Start
 *       7 is not legal, so node 1 is not in A; a minimum over every node would stay at node 1's 0 and refuse member 2.
 *
 * Every gang kind node-scored (ISL_FLAG_GANG_NODE_SCORE_ALL): a cluster that packs with MostAllocated or spreads with LeastAllocated runs
 * its elastic jobs, its jobs that prefer few nodes and its balanced replicas on the same engine as its pods.  Each kind keeps its own
 * first criterion (a few-node round's largest d, an elastic one-node trim's depth D, a balanced member's candidate nodes); the node score
 * breaks the ties below it where a first-fit engine takes scan order.  On an engine created with the flag:
 *   C1. isl_create: ISL_EINVAL for the flag without ISL_FLAG_GANG_NODE_SCORE (hence without a node-scoring policy).  With both bits the
 *       engine also accepts ISL_FLAG_GANG_FEW_NODES (N1's refusal is lifted; F6's refusal with ISL_FLAG_GANG_ONE_NODE, _DISTINCT_NODES and
 *       _LOCALITY stays), ISL_FLAG_GANG_MIN_MEMBERS (the refusals of N1 and M6 are lifted) and ISL_FLAG_GANG_BALANCED with
 *       ISL_FLAG_GANG_LOCALITY (B6's refusal of node scoring is lifted).  Every other refusal stays: ISL_FLAG_ALL_NODES,
 *       ISL_FLAG_GANG_PREEMPT with few-node or elastic gangs (P7), BALANCED without LOCALITY, two locality flags, and node scoring's
 *       ISL_ERANGE above 2^20 GPUs or nodes.  An engine without the bit keeps every code it returns.
 *   C2. Under ISL_FLAG_GANG_LOCALITY a byte of 2 is accepted (N6 is lifted), and under ISL_FLAG_GANG_BALANCED so are 4..255.  Every other
 *       check of L4 and M6 is unchanged and still runs before the engine state is looked at.
 *   C3. score_N(R) is node-scoring rule 3 over N's GPUs inside the partition with N's table width: MostAllocated floor(100 (busy + R) /
 *       cap), LeastAllocated floor(100 (cap - busy - R) / cap), busy counted on the occupancy the round or member sees (the call's FREEs,
 *       the committed gangs and the gang's own tentative members).  Ties go to the lowest canonical node index; inside a node the
 *       reference's first-fit search decides, as in N5.
 *   C4. Few nodes (ISL_FLAG_GANG_FEW_NODES, or byte 2): F2's rounds and d(N) are unchanged; among the nodes with the largest d >= 1 the
 *       round goes to the highest score_N(R_d(N)), R_d(N) the sum of the row sizes, in N's table, of the d members the node takes.  F3's
 *       failure and rule 5 are unchanged.  Consequences: (a) a gang that some node takes whole gets exactly N5's records and occupancy;
 *       (b) a gang that fails here fails on the one-node scored engine in the same state; (c) on a one-node inventory, or a partition
 *       inside one node, a call equals a FIRST_FIT engine with the few-node flag; (d) with gangs of one a call equals isl_place_batch on
 *       the same engine; (e) F4 (e) holds: two consecutive rounds never use the same node.
 *   C5. Elastic gangs (ISL_FLAG_GANG_MIN_MEMBERS): M1-M7 hold with the scored rules as the rules of each locality: N3 any node, N4
 *       distinct nodes, N5 one node, C4 few nodes, C6 balanced.  M3 trims member by member for any-node, distinct-node and balanced gangs
 *       and after the rounds so far for few-node gangs; a one-node gang commits its first D members on the node that reaches depth D with
 *       the highest score_N(R_D(N)).  M5 (a)-(d) hold: a gang trimmed at f equals the cut gang of f members placed without the flag.
 *   C6. Balanced gangs (bytes 4..255): B2's A, cnt, mu and candidate nodes (cnt <= mu + k - 1) are unchanged; among the candidates the
 *       member goes to the highest score_N(its row size).  B3, B5, B7 and B8 hold, and B4 (a)-(f) with N4 in place of S2 and N3 in place
 *       of rules 2-4: byte 3 + k with k >= the gang's ALLOC members equals byte 0, which is N3.
 *   C7. With the bit, a call whose gangs all have locality 0, 1 or 3, without ISL_FLAG_GANG_MIN_MEMBERS, returns exactly what the same
 *       engine without the bit returns (records, occupancy, stats.placed).  Every other entry point returns what it returns without the
 *       bit; isl_preempt keeps P1, so bytes 2 and above 3 are ISL_EINVAL there.
 *   C8. The score never comes above the locality's own criterion: a round never takes fewer members for a better score and a trim never
 *       keeps fewer members.  The choice stays greedy, as F5, S4, B7 and M7 say.
 *   Examples, H100-80GB rows, either quirk set, one-GPU nodes, gangs of four 1g.10gb, records (gpu, start):
 *       few nodes, bytes 0x0F 0xF8 0x3F   FIRST_FIT (F2): d = [3, 3, 1], node 0 takes (0,4) (0,5) (0,6); then d = [0, 1, 1]: (1,0).
 *                                         MOST: round 1 scores node 0 87, node 1 100: (1,0) (1,1) (1,2); round 2 node 0 62, node 2 87:
 *                                         (2,6).  LEAST: round 1 node 0 12, node 1 0: (0,4) (0,5) (0,6); round 2 node 1 25, node 2 12:
 *                                         (1,0).
 *       one node, m = 2, same nodes       D = 3, reached by nodes 0 and 1.  MOST (1,0) (1,1) (1,2); LEAST (0,4) (0,5) (0,6); member 3
 *                                         NO_CAPACITY either way.
 *       balanced, bytes 0x00 0x0F         byte 4: LEAST (0,0) (1,4) (0,1) (1,5), MOST (1,4) (0,0) (1,5) (0,1);
 *                                         byte 5: LEAST (0,0) (0,1) (1,4) (0,2), MOST (1,4) (1,5) (0,0) (1,6).
 */
int  isl_place_gangs(isl_engine* e, uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out);

/* 8 bytes: one running allocation that MAY be evicted (isl_preempt). */
typedef struct isl_victim {
    uint32_t gpu;                  /* canonical GPU index */
    uint8_t  start, size;          /* its span */
    uint8_t  priority;             /* rank, higher = more important; 255 = never evicted */
    uint8_t  pad;
} isl_victim;

/* Priority preemption (the kube-scheduler's PriorityClass preemption for pods the scheduler never sees): for each pending pod that
 * does not fit, which GPU and start it should take and which lower-priority allocations must leave first.  `in`, `priority` (one byte
 * per request, higher = more important), `out` and `evict` (n x 8 uint32) are host buffers of n entries; `victims` has n_victims.
 *   1. A query.  The live occupancy, a snapshot (isl_snapshot_occupancy), the partition and the stats (except kernel_launches) are the
 *      same after the call as before; everything runs under one engine lock.  The caller deletes the victim pods; once their
 *      Allocations entries are gone, an ordinary placement call places the pod.
 *   2. Each victims[k] names a span that is busy in the live occupancy.  Every busy slice not covered by a listed victim is pinned
 *      (dangling Prepared slices, allocations the caller does not list, victims with priority 255).  A victim on a GPU outside the
 *      engine's partition is ignored, as isl_free_batch ignores such spans.  ISL_EINVAL, nothing changed: a victim with size 0,
 *      start + size > 8 or gpu >= G, or (inside the partition) one that covers a free slice or overlaps another victim.
 *   3. The preemptors are in[i] at priority[i], in array order; preemptor i sees the state left by 0..i-1 of the same call: their
 *      victims are gone (slices free, no longer listed), their own spans busy and pinned.  An ALLOC of an unknown profile gets the
 *      BAD_PROFILE record of isl_place_batch; ISL_OP_FREE makes the call ISL_EINVAL (the victim list is how releases are expressed);
 *      any other op gets an ISL_ST_NOOP record.
 *   4. A candidate for an ALLOC of profile p at priority pi is a GPU g of the partition with a start v of p's row in the table of g's
 *      node, legal under the engine's quirk set (candidate_mask, the rule of the start search), such that every busy slice of the
 *      mask belongs to a listed victim with priority < pi.  V(g, v) is every victim that overlaps the mask; a victim leaves whole,
 *      also where it extends beyond the mask.
 *   5. The choice is the lexicographic minimum over all candidates of: the highest priority in V (an empty V below every priority),
 *      the sum of V's priorities, |V|, the GPU's position in the engine's scan order (ascending canonical index; descending under
 *      ISL_POLICY_RIGHT_TO_LEFT; ascending for the best-fit family and node scoring), v's position in the row — the order of the kube-scheduler's
 *      pickOneNodeForPreemption without its PodDisruptionBudget and start-time keys.  The record is PLACED (g, v, size) and
 *      evict[8i .. 8i+8) holds the indices into `victims` of V in ascending order, padded with ISL_GPU_NONE.  With no candidate the
 *      record is the usual unplaced one (NO_CAPACITY, gpu NONE, start 9, the default size); a record that is not PLACED has an
 *      evict row of ISL_GPU_NONE only.  Consequences:
 *      (a) v is what the start search (:343-383) returns on g's occupancy with V removed: an earlier start in the row would need a
 *          subset of V, and so would have a smaller key.
 *      (b) a pod that fits without eviction evicts nothing: a one-request call on a FIRST_FIT or RIGHT_TO_LEFT engine returns the
 *          record isl_place_batch returns.
 *   6. Every policy, both quirk sets, per-node tables, inside isl_set_partition.  n == 0 does nothing.
 *      ISL_EINVAL: NULL buffers with n > 0 (or victims NULL with n_victims > 0), an engine created with ISL_FLAG_ALL_NODES.
 *      ISL_ERANGE: n > max_batch, n_victims > 8 x max_gpus, a partition that is empty or holds more than 2^20 GPUs.
 *      ISL_ESTATE: no profiles or inventory, or an open stream.
 *
 * Gang preemption (ISL_FLAG_GANG_PREEMPT): a high-priority job whose pods must all run, or none of them (a gang of isl_place_gangs), asks
 * for the victims of the whole gang in one query, so that no pod is deleted for a gang that still cannot run.  On an engine created with
 * the flag, rules 1-6 hold except where these say otherwise:
 *   P1. Gangs.  A gang is a maximal run of consecutive requests with equal `handle` (opaque otherwise, never echoed).  Its ALLOC members
 *       carry the same `priority` byte, the gang's priority.  Its locality is the engine's: one node under ISL_FLAG_GANG_ONE_NODE,
 *       distinct nodes under ISL_FLAG_GANG_DISTINCT_NODES, under ISL_FLAG_GANG_LOCALITY the ALLOC members' `start` byte as in L1 (0, 1
 *       or 3), else any node.  ISL_EINVAL, nothing changed, when two ALLOC members of one gang carry different priority bytes, or under
 *       ISL_FLAG_GANG_LOCALITY different locality bytes, or a locality byte of 2 (few nodes) or above 3; these checks run with the other
 *       argument checks, before the engine state is looked at (as L4 and M6).  A FREE is still ISL_EINVAL (rule 3).  Other ops report
 *       NOOP with an all-NONE evict row and do not count.
 *   P2. Order.  Gangs go in array order.  Gang i sees the state the COMMITTED gangs before it left: their victims gone, their spans busy
 *       and pinned.  An aborted gang leaves no trace.
 *   P3. Choice.  Any node: the ALLOC members in order, each chosen by rules 4-5 over the partition, each seeing the gang's earlier
 *       members (their victims gone, their spans pinned).  Distinct nodes: the same, restricted to the GPUs whose node holds no earlier
 *       member of the gang (a node the partition cuts counts as one node, as in S2).  One node: for every node N of the partition the
 *       members are resolved in order by rules 4-5 restricted to N's GPUs inside the partition; N can take the gang when every member
 *       gets a candidate, and its cost is the lexicographic tuple (the highest priority among all the victims the members evict + 1, or
 *       0 with none; the sum of their priorities; how many they are; N's position in the engine's scan order of rule 5).  The gang goes
 *       to the node of least cost: pickOneNodeForPreemption with the gang treated as one pod.
 *   P4. Commit.  Every ALLOC member gets a PLACED record (gpu, start, size), and its evict row the victims it evicts, ascending, padded
 *       with ISL_GPU_NONE.  The union of a gang's rows is what the caller deletes.
 *   P5. Failure.  Any node and distinct nodes: rule 4 of isl_place_gangs (the first member without a candidate keeps its NO_CAPACITY or
 *       BAD_PROFILE record, every other ALLOC member reports ISL_ST_GANG_ABORTED).  One node: G3, with D the largest number of leading
 *       ALLOC members that any node resolves with evictions.  Every evict row of an aborted gang is all ISL_GPU_NONE.
 *   P6. Consequences.  (a) With all handles distinct (gangs of one) a flagged call equals the unflagged one under every policy, quirk
 *       set, locality, node table and partition, records and evict rows (for one-node gangs of one because a node's GPUs are contiguous
 *       in scan order).  (b) With no victim listed, or none below its gang's priority, a flagged FIRST_FIT or RIGHT_TO_LEFT call returns
 *       the records isl_place_gangs returns on the same engine and requests, for localities 0, 1 and 3.  (c) The call is a query (rule 1).
 *       (d) With the victims of a committed gang, and of every committed gang before it, removed, the gang's spans are free and pairwise
 *       disjoint; a one-node gang's members share one node (isl_gpu_to_node), a distinct-node gang's members are on distinct nodes.
 *       (e) Under any-node locality a call equals its gangs run one at a time through the unflagged isl_preempt, each gang's evictions
 *       and spans applied when every member was placed and dropped otherwise.
 *   P7. isl_create: ISL_EINVAL for the flag with ISL_FLAG_ALL_NODES, ISL_FLAG_GANG_FEW_NODES or ISL_FLAG_GANG_MIN_MEMBERS.  A
 *       node-scoring engine takes it, with any-node gangs (its locality flags are refused already).  isl_preempt keeps every code of
 *       rule 6, the 2^20-GPU partition cap included.  Every other entry point, isl_place_gangs included, returns exactly what it returns
 *       without the flag.
 *   P8. Greedy, member by member (as S4 and F5): a gang can abort although some choice of victims would fit it.  A100-40GB rows,
 *       reference-exact quirks, first-fit, one GPU with byte 0x01 held by a victim of priority 0, a gang of priority 1: [1g.5gb, 4g.20gb]
 *       aborts (the 1g takes the free start 1, since an empty V wins, and pins a slice the 4g needs), [4g.20gb, 1g.5gb] commits (the 4g
 *       takes start 0 and evicts the victim, the 1g takes start 4).  List the larger members first. */
int  isl_preempt(isl_engine* e, uint32_t n, const isl_request* in, const uint8_t* priority,
                 uint32_t n_victims, const isl_victim* victims, isl_result* out, uint32_t* evict);

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
 * overlap on the device (segment pipeline).  While a stream is open (isl_stream_open until isl_stream_close, launched or not) every
 * call on the engine returns ISL_ESTATE and changes nothing, except: isl_stream_submit, _wait and _close, isl_destroy (closes the stream
 * first), and isl_num_gpus, isl_gpu_to_node, isl_device_occupancy, isl_device_results, isl_abi_version, isl_strerror,
 * isl_last_cuda_error, isl_host_alloc and isl_host_free.  The test is made under the engine lock.
 * isl_stream_open returns ISL_ERANGE, and leaves no stream open, when max_batches x 65 536 > max_batch, or when the inventory does not
 * fit one resident pipeline beside the feed kernels: the pipeline then has SMs - 4 stages of at most 8 x 512 GPUs, so on a 132-SM H100
 * an inventory of more than 128 x 8 x 512 = 524 288 GPUs (fewer when the loaded tables cap the sub-segment below 512 GPUs) is refused.
 * isl_place_stream takes the chunk-by-chunk path for such inventories instead. */
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
 *      never repeated stream_id (it tags what crosses the ranks); only enqueues.  Results: element-wise MIN over ranks as for the batch variant.
 *      The speculative rounds (isl_connect_spec_local / isl_ipc_connect_spec) tag their records with the low 24 bits of the id, and the
 *      shared record memory is cleared only when it is allocated, so that ids s and s + 2^24 would share a tag: only a stream id below
 *      2^24 speculates; a larger one takes the token ring (same records, all ranks decide alike).  An engine whose record memory is
 *      shared (isl_ipc_spec_handle, isl_connect_spec_local, also after a disconnect) never speculates outside
 *      isl_place_stream_partitioned: isl_place_stream, isl_place_batch and open streams on it keep the plain pipeline. */
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
