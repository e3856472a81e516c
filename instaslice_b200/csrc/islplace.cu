// islplace.cu — C ABI (include/islplace.h) and host-side orchestration of the placement engine.
//
// The entry points replace, for the allocator path only, what the Go controller does in
// internal/controller/instaslice_controller.go:188-262,303-384 (see the header for the per-symbol map).
// No Go pointer is retained after a call returns; every buffer the engine keeps is its own.
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <mutex>
#include <new>
#include <optional>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "isl_kernels.cuh"

using namespace isl;

static constexpr uint32_t kMaxStreamChunks = 4096;
static constexpr uint32_t kSpecRingIds = 1u << 24;     // stream ids of isl_place_stream_partitioned that may speculate

// One instantiation of k_ganglocal or k_preempt_gangs: the template arguments it was built with and the name a launch error carries.
struct GangKernel {
    const void* fn;
    const char* name;
    uint32_t loc;                    // kLoc: an ISL_GANG_* byte for every gang, or kLocPerGang
    bool min, score, bal;            // kMin, kScore, kBal of k_ganglocal; false for k_preempt_gangs
};
const GangKernel kGangKernels[] = {
    {(const void*)k_ganglocal<ISL_GANG_ONE_NODE>, "k_ganglocal<one_node>", ISL_GANG_ONE_NODE, false, false, false},
    {(const void*)k_ganglocal<ISL_GANG_FEW_NODES>, "k_ganglocal<few_nodes>", ISL_GANG_FEW_NODES, false, false, false},
    {(const void*)k_ganglocal<ISL_GANG_DISTINCT_NODES>, "k_ganglocal<distinct_nodes>", ISL_GANG_DISTINCT_NODES, false, false, false},
    {(const void*)k_ganglocal<kLocPerGang, false>, "k_ganglocal<per_gang>", kLocPerGang, false, false, false},
    {(const void*)k_ganglocal<kLocPerGang, true>, "k_ganglocal<per_gang, min_members>", kLocPerGang, true, false, false},
    {(const void*)k_ganglocal<ISL_GANG_ANY_NODES, false, true>, "k_ganglocal<any_node, node_score>", ISL_GANG_ANY_NODES, false, true, false},
    {(const void*)k_ganglocal<ISL_GANG_ONE_NODE, false, true>, "k_ganglocal<one_node, node_score>", ISL_GANG_ONE_NODE, false, true, false},
    {(const void*)k_ganglocal<ISL_GANG_DISTINCT_NODES, false, true>, "k_ganglocal<distinct_nodes, node_score>", ISL_GANG_DISTINCT_NODES, false, true, false},
    {(const void*)k_ganglocal<kLocPerGang, false, true>, "k_ganglocal<per_gang, node_score>", kLocPerGang, false, true, false},
    {(const void*)k_ganglocal<kLocPerGang, false, false, true>, "k_ganglocal<per_gang, balanced>", kLocPerGang, false, false, true},
    {(const void*)k_ganglocal<kLocPerGang, true, false, true>, "k_ganglocal<per_gang, min_members, balanced>", kLocPerGang, true, false, true},
    {(const void*)k_ganglocal<ISL_GANG_FEW_NODES, false, true>, "k_ganglocal<few_nodes, node_score>", ISL_GANG_FEW_NODES, false, true, false},
    {(const void*)k_ganglocal<kLocPerGang, true, true>, "k_ganglocal<per_gang, min_members, node_score>", kLocPerGang, true, true, false},
    {(const void*)k_ganglocal<kLocPerGang, false, true, true>, "k_ganglocal<per_gang, node_score, balanced>", kLocPerGang, false, true, true},
    {(const void*)k_ganglocal<kLocPerGang, true, true, true>, "k_ganglocal<per_gang, min_members, node_score, balanced>", kLocPerGang, true, true, true},
};
const GangKernel kPreemptGangKernels[] = {
    {(const void*)k_preempt_gangs<ISL_GANG_ANY_NODES>, "k_preempt_gangs<any_node>", ISL_GANG_ANY_NODES, false, false, false},
    {(const void*)k_preempt_gangs<ISL_GANG_ONE_NODE>, "k_preempt_gangs<one_node>", ISL_GANG_ONE_NODE, false, false, false},
    {(const void*)k_preempt_gangs<ISL_GANG_DISTINCT_NODES>, "k_preempt_gangs<distinct_nodes>", ISL_GANG_DISTINCT_NODES, false, false, false},
    {(const void*)k_preempt_gangs<kLocPerGang>, "k_preempt_gangs<per_gang>", kLocPerGang, false, false, false},
};

// What kind of gang engine a config makes, decoded once by isl_create from its flags and policy (gang_mode).
struct GangMode {
    uint32_t locality = ISL_GANG_ANY_NODES;      // an ISL_GANG_* byte for every gang, or kLocPerGang (ISL_FLAG_GANG_LOCALITY)
    bool min_members = false, node_score = false, score_all = false, balanced = false;
    bool gangs_refused = false;                  // isl_place_gangs refuses every call
    const GangKernel* place = nullptr;           // the k_ganglocal isl_place_gangs launches; none: k_bestfit's gang loop
    const GangKernel* preempt = nullptr;         // the k_preempt_gangs isl_preempt launches; none: k_preempt, gangs of one
};

// What plan_pipeline decides for one k_pipeline launch: GPUs per stage (seg), stages, GPUs per sub-segment, speculative rounds.
struct PipePlan {
    uint32_t seg = 0, n_seg = 0, sub = 0;
    bool spec = false;
};

// Owners of the engine's CUDA resources.  Each is move-only and releases its resource in its destructor, so deleting an isl_engine
// (with its device current) frees everything it holds.  They convert to the raw pointer or handle for kernel arguments and CUDA calls.
enum class Growth { exact, headroom };       // headroom: need + need / 4 + 1 units, so that a growing stream reallocates rarely

// Device memory of cap() units of `unit` elements each.
template <typename T>
class DevMem {
    T* p_ = nullptr; size_t cap_ = 0, unit_;
  public:
    explicit DevMem(size_t unit = 1) : unit_(unit) {}
    DevMem(DevMem&& o) noexcept : p_(std::exchange(o.p_, nullptr)), cap_(std::exchange(o.cap_, 0)), unit_(o.unit_) {}
    ~DevMem() { release(); }
    operator T*() const { return p_; }
    T* get() const { return p_; }
    size_t cap() const { return cap_; }
    size_t bytes() const { return cap_ * unit_ * sizeof(T); }
    void release() { if (p_) cudaFree(p_); p_ = nullptr; cap_ = 0; }
    // Room for `need` units.  A buffer that is too small is freed and allocated anew (*fresh: it was, its contents are undefined); a
    // failed allocation leaves it empty.
    cudaError_t reserve(size_t need, Growth g = Growth::exact, bool* fresh = nullptr) {
        if (fresh) *fresh = false;
        if (need <= cap_) return cudaSuccess;
        release();
        const size_t units = g == Growth::headroom ? need + need / 4 + 1 : need;
        if (cudaError_t err = cudaMalloc(&p_, units * unit_ * sizeof(T))) { p_ = nullptr; return err; }
        cap_ = units;
        if (fresh) *fresh = true;
        return cudaSuccess;
    }
    cudaError_t replace(size_t n) { release(); return reserve(n); }      // exactly n units, whatever the buffer held
};

// Pinned host memory of cap() elements; a mapped buffer (cudaHostAllocMapped) also holds its device alias dev().
template <typename T>
class HostMem {
    T *p_ = nullptr, *dev_ = nullptr;
    size_t cap_ = 0; unsigned flags_;
  public:
    explicit HostMem(unsigned flags) : flags_(flags) {}
    HostMem(HostMem&& o) noexcept : p_(std::exchange(o.p_, nullptr)), dev_(std::exchange(o.dev_, nullptr)), cap_(std::exchange(o.cap_, 0)), flags_(o.flags_) {}
    ~HostMem() { release(); }
    operator T*() const { return p_; }
    T* dev() const { return dev_; }
    void release() { if (p_) cudaFreeHost(p_); p_ = dev_ = nullptr; cap_ = 0; }
    // Room for n elements, exactly.  A buffer that is too small is freed first; a failed allocation leaves it empty.
    cudaError_t reserve(size_t n) {
        if (n <= cap_) return cudaSuccess;
        release();
        cudaError_t err = cudaHostAlloc(&p_, n * sizeof(T), flags_);
        if (err != cudaSuccess) { p_ = nullptr; return err; }
        if (flags_ & cudaHostAllocMapped) err = cudaHostGetDevicePointer(&dev_, p_, 0);
        if (err == cudaSuccess) cap_ = n; else release();
        return err;
    }
};

// A stream, event or peer mapping, released (Release) only if this holder owns it: out() is where a create or open call writes a
// handle the holder then owns; borrow() keeps one that belongs to someone else (a caller's stream, a same-process engine's memory,
// the engine's own record memory).
template <typename H, auto Release>
class Handle {
    H h_ = nullptr; bool own_ = false;
  public:
    Handle() = default;
    Handle(Handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)), own_(std::exchange(o.own_, false)) {}
    ~Handle() { reset(); }
    operator H() const { return h_; }
    H get() const { return h_; }
    void reset() { if (own_ && h_) Release(h_); h_ = nullptr; own_ = false; }
    void borrow(H h) { reset(); h_ = h; }
    H* out() { reset(); own_ = true; return &h_; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;
template <typename T> using PeerMap = Handle<T*, cudaIpcCloseMemHandle>;      // opened through CUDA IPC, or borrowed

struct isl_engine {
    // declared first, so destroyed last: the memory below is freed before the streams it was used on go away
    Stream stream;
    // host-buffer streams: batches are fed on their own stream while the pipeline runs; results leave chunk by chunk
    Stream feed_stream; Event ev_feed, ev_feed_done;
    Event ev[6];                     // ISL_FLAG_TIMING
    isl_config cfg{};
    int device = 0;
    std::mutex mu;
    char cuda_err[256] = {0};

    DevProfiles prof{};
    bool have_profiles = false, have_inventory = false;
    CandTab tab{};
    uint32_t n_cand_slots = 0;       // K of k_chain<K>
    uint32_t cand_profiles = 0;      // profiles with >= 1 valid (profile, start) candidate

    uint32_t G = 0, lo = 0, hi = 0;
    std::vector<uint32_t> node_off;
    // per-node profile tables (heterogeneous clusters): rows_all[t][p], n_starts == 0 = table t has no row of name p
    uint32_t n_tables = 1;
    isl_profile rows_all[ISL_MAX_TABLES][ISL_MAX_PROFILES] = {};
    std::vector<uint8_t> node_table;     // table of every node (empty = all 0)
    DevMem<uint8_t> d_gtab;              // table of every GPU's node, one byte per GPU
    DevMem<uint8_t> d_capn;              // [table][profile][occ]: placements of the profile the GPU takes in a row
    DevMem<uint32_t> d_seq;              // [table][profile][occ]: their starts, 4 bits each
    DevMem<uint8_t> d_sizes;             // [table][profile]: slices per placement
    DevMem<uint8_t> d_score;             // [profile][occ] of table 0: what a best-fit family policy minimises (k_bestfit)
    DevMem<unsigned long long> d_cap;    // isl_capacity: per-profile counters
    DevMem<uint16_t> d_cand_o16;         // single-chain path: occupancy + table tag of every candidate

    // device buffers
    DevMem<uint8_t> d_occ;           // one byte per GPU, padded to whole sweep blocks with 0xFF
    size_t occ_bytes = 0;
    DevMem<uint8_t> d_lut;           // [16][256]
    DevMem<uint16_t> d_feas;         // [256]
    DevMem<uint2> d_req;             // staging for the host-buffer entry point
    DevMem<uint2> d_res;             // results, then kMaxStreamChunks 'ranks done' counters of a partitioned run (peer-mapped with them)
    DevMem<uint16_t> d_q;            // per-chunk queues
    DevMem<uint32_t> d_tile_counts;
    DevMem<uint32_t> d_cand;
    DevMem<uint2> d_log;             // decision log of one chunk (chain -> commit)
    DevMem<uint32_t> d_bf_bitmaps;   // best-fit class bitmaps for inventories beyond the shared-memory size / several tables
    HostMem<uint2> h_small_out{cudaHostAllocMapped};     // results of tiny batches (k_small writes them over PCIe directly)
    DevMem<uint32_t> d_sweep_counts;
    DevMem<Ctrl> d_ctrl;
    DevMem<uint8_t> d_scratch;       // eval_starts / free_batch / gang offsets staging
    // stream / segment-pipeline state (grown on demand)
    DevMem<ChunkDesc> d_chunks; DevMem<Ctrl> d_cctl; DevMem<uint16_t> d_qall; DevMem<uint32_t> d_tokens{kTokStride};
    DevMem<uint32_t> d_free_acc; DevMem<TileDesc> d_tiles; std::vector<TileDesc> h_tiles;
    uint32_t pipe_chunk = 0;         // requests per pipeline chunk (multiple of kTile, <= kChunk)
    std::vector<ChunkDesc> h_chunks;
    uint32_t epoch = 0;
    DevMem<uint32_t> d_inbox{kTokStride};   // [kMaxStreamChunks][kTokStride] tokens written by the previous rank (peer store)
    PeerMap<uint32_t> d_outbox;      // next rank's inbox
    bool has_prev = false;
    DevMem<unsigned long long> d_trace{kTraceWords}; uint32_t trace_chunks = 0, trace_seg = 0;
    int max_coresident = 0;          // CTAs of k_pipeline that can be resident at once (0 = not queried)
    DevMem<uint32_t> d_ready;        // [batch] epoch flag
    DevMem<uint32_t> d_done_cnt;     // [chunk] committed segments
    DevMem<uint8_t> d_occ_snap; uint32_t snap_G = 0;      // isl_snapshot_occupancy / isl_restore_occupancy
    // isl_preempt: the victim-index map (8 words per GPU of the partition), the victims, staging of [candidate masks | priorities], the
    // evict rows, the per-CTA minima of k_preempt and k_victim_map's error word.  ISL_FLAG_GANG_PREEMPT (k_preempt_gangs): the gang
    // offsets followed by the locality bytes, the rollback log (one entry per request), the per-GPU state when the shares do not fit in
    // shared memory, and the dynamic shared memory one CTA of the engine's instantiation may have
    struct Preempt {
        DevMem<uint32_t> vmap, evict, err, gangs;
        DevMem<isl_victim> victims;
        DevMem<uint8_t> stage, state;
        DevMem<unsigned long long> keys;
        DevMem<PgLog> log;
        int optin = 0;
    } pre;
    // node scoring (k_nodefit): the inventory's node offsets (isl_load_inventory), the per-profile min-trees when they do not fit in shared
    // memory, the per-(profile, node) fit counts and the per-node busy / cap words, grown to the partition; the width of every table
    struct NodeFit {
        DevMem<uint32_t> node_off, tree, fit, nodes;
        uint8_t width[kMaxTables] = {};
    } nf;
    // gang topology (gang.place, k_ganglocal): the inventory's node offsets in storage order (host and device, isl_load_inventory), the
    // scratch copies or node-used marks when the shares do not fit in shared memory, the per-CTA minima, and the per-CTA stacks of wins
    // of distinct-node gangs
    struct GangNode {
        std::vector<uint32_t> off;
        DevMem<uint32_t> node_off;
        DevMem<uint8_t> scratch;
        DevMem<unsigned long long> keys;
        DevMem<uint2> wins;
        int optin = 0;               // dynamic shared memory one CTA of gang.place may have
    } gn;
    GangMode gang;
    unsigned long long wait_ns = 20000000000ull;   // a starved device-side wait traps after this long (ISL_WAIT_SECONDS overrides the 20 s)
    uint32_t window = 0;             // causal window of stream calls (isl_set_causal_window): chunk c starts after chunk c - window is committed
    uint32_t spec_mode = ISL_SPEC_AUTO;     // speculative rounds (isl_set_speculation); ISL_SPEC=0|1 in the environment overrides
    DevMem<unsigned long long> d_specdbg{8};      // [kSpecRounds][8]
    DevMem<unsigned long long> d_spec{kSpecWordsPerChunk}; uint32_t spec_hi = 0;    // record memory of the rounds, cap() chunks
    // partitioned inventory: every rank's record memory, peer-mapped (own entry = d_spec); bounds of all ranks; the shared memory never moves
    PeerMap<unsigned long long> spec_peer[8]; bool spec_shared = false;
    uint32_t spec_world = 0, spec_rank = 0, spec_bounds[9] = {};
    // open stream (isl_stream_open / _submit / _wait / _close): one persistent k_pipeline, batches arrive while it runs
    struct Open {
        bool active = false, launched = false;
        uint32_t max_batches = 0, submitted = 0, epoch = 0, q_stride = 0, free_stride = 0, tiles_per_batch = 0;
        PipePlan plan;
        HostMem<uint32_t> h_done{cudaHostAllocMapped};        // [batch] = epoch once its results are in host memory
        HostMem<ChunkDesc> h_chunks{cudaHostAllocDefault};    // staging of the per-batch descriptors
        HostMem<TileDesc> h_tiles{cudaHostAllocDefault};
    } open;
    // partitioned inventory with the results gathered on the owner rank (rank 0): peer-mapped d_res of the owner
    PeerMap<uint2> d_owner_out;
    uint32_t ring_world = 0;         // ranks of the partitioned run (isl_set_ring_world); the causal window of a ring needs it

    // stats
    isl_stats st{};
};

namespace {

inline bool bestfit_family(uint32_t policy) { return policy == ISL_POLICY_BEST_FIT || policy == ISL_POLICY_MIN_FRAG; }
inline bool node_scoring(uint32_t policy) { return policy == ISL_POLICY_MOST_ALLOCATED || policy == ISL_POLICY_LEAST_ALLOCATED; }
// The engines whose batches one CTA resolves request by request (k_bestfit, k_nodefit): the best-fit family, node scoring, and every
// policy under ISL_FLAG_FIRST_AVAILABLE (a pod's fallback sees the occupancy its predecessors left).  No latency kernels, no segment
// pipeline, no partitioned calls or open streams, at most kBfMaxGpus GPUs
inline bool request_major(const isl_config& cfg) {
    return bestfit_family(cfg.policy) || node_scoring(cfg.policy) || (cfg.flags & ISL_FLAG_FIRST_AVAILABLE);
}
inline bool first_available(const isl_engine* e) { return e->cfg.flags & ISL_FLAG_FIRST_AVAILABLE; }
inline bool reversed(const isl_engine* e) { return e->cfg.policy == ISL_POLICY_RIGHT_TO_LEFT; }

// The entry of `table` built with these template arguments, nullptr when none is
template <size_t N>
const GangKernel* find_gang_kernel(const GangKernel (&table)[N], uint32_t loc, bool min, bool score, bool bal) {
    for (const GangKernel& k : table)
        if (k.loc == loc && k.min == min && k.score == score && k.bal == bal) return &k;
    return nullptr;
}

// The gang mode of a config with a valid policy, or ISL_EINVAL for a combination of gang flags and policy isl_create refuses: the
// rules of G5, S6, F6, L5, M6, P7, N1, B6 and C1 in include/islplace.h.  Elastic gangs read each gang's byte, so they run the per-gang
// k_ganglocal, whose bytes isl_place_gangs fills with the engine's locality when the gangs do not name it.
int gang_mode(const isl_config* cfg, GangMode* m) {
    const uint32_t f = cfg->flags;
    const bool scoring = node_scoring(cfg->policy);
    auto has = [f](uint32_t bits) { return (f & bits) != 0; };
    const uint32_t localities = f & (ISL_FLAG_GANG_ONE_NODE | ISL_FLAG_GANG_DISTINCT_NODES | ISL_FLAG_GANG_FEW_NODES | ISL_FLAG_GANG_LOCALITY);
    const uint32_t gang_flags = ISL_FLAG_GANG_ONE_NODE | ISL_FLAG_GANG_DISTINCT_NODES | ISL_FLAG_GANG_FEW_NODES | ISL_FLAG_GANG_LOCALITY |
                                ISL_FLAG_GANG_MIN_MEMBERS | ISL_FLAG_GANG_PREEMPT | ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_BALANCED |
                                ISL_FLAG_GANG_NODE_SCORE_ALL;
    if (localities & (localities - 1)) return ISL_EINVAL;                       // at most one locality flag
    if (has(ISL_FLAG_ALL_NODES) && has(gang_flags)) return ISL_EINVAL;           // a pod on every node: no gang kind applies
    if (has(ISL_FLAG_GANG_NODE_SCORE_ALL) && !has(ISL_FLAG_GANG_NODE_SCORE)) return ISL_EINVAL;
    if (has(ISL_FLAG_GANG_NODE_SCORE) && !scoring) return ISL_EINVAL;
    // under node scoring a gang kind takes the node score, or is refused
    if (scoring && has(ISL_FLAG_GANG_ONE_NODE | ISL_FLAG_GANG_DISTINCT_NODES | ISL_FLAG_GANG_LOCALITY) && !has(ISL_FLAG_GANG_NODE_SCORE))
        return ISL_EINVAL;
    if (scoring && has(ISL_FLAG_GANG_FEW_NODES | ISL_FLAG_GANG_MIN_MEMBERS | ISL_FLAG_GANG_BALANCED) && !has(ISL_FLAG_GANG_NODE_SCORE_ALL))
        return ISL_EINVAL;
    if (has(ISL_FLAG_GANG_BALANCED) && !has(ISL_FLAG_GANG_LOCALITY)) return ISL_EINVAL;        // the maxSkew is a locality byte
    if (has(ISL_FLAG_GANG_PREEMPT) && has(ISL_FLAG_GANG_FEW_NODES | ISL_FLAG_GANG_MIN_MEMBERS)) return ISL_EINVAL;     // no preemption order
    m->locality = has(ISL_FLAG_GANG_LOCALITY)        ? kLocPerGang
                  : has(ISL_FLAG_GANG_ONE_NODE)      ? ISL_GANG_ONE_NODE
                  : has(ISL_FLAG_GANG_FEW_NODES)     ? ISL_GANG_FEW_NODES
                  : has(ISL_FLAG_GANG_DISTINCT_NODES) ? ISL_GANG_DISTINCT_NODES
                                                      : ISL_GANG_ANY_NODES;
    m->min_members = has(ISL_FLAG_GANG_MIN_MEMBERS);
    m->node_score = has(ISL_FLAG_GANG_NODE_SCORE);
    m->score_all = has(ISL_FLAG_GANG_NODE_SCORE_ALL);
    m->balanced = has(ISL_FLAG_GANG_BALANCED);
    m->gangs_refused = has(ISL_FLAG_ALL_NODES) || (scoring && !m->node_score);
    // every mode the rules accept has its instantiations; one without would be refused here, never run on another kernel
    if ((m->locality != ISL_GANG_ANY_NODES || m->min_members || m->node_score) &&
        !(m->place = find_gang_kernel(kGangKernels, m->min_members ? kLocPerGang : m->locality, m->min_members, m->node_score, m->balanced)))
        return ISL_EINVAL;
    if (has(ISL_FLAG_GANG_PREEMPT) && !(m->preempt = find_gang_kernel(kPreemptGangKernels, m->locality, false, false, false))) return ISL_EINVAL;
    return ISL_OK;
}

// The byte field(r) that every ALLOC request r of in[r0, r1) carries, in *v (left as it was when none is an ALLOC): the number of ALLOC
// requests, or -1 when two of them differ.
template <typename Field>
int64_t alloc_shared(const isl_request* in, uint32_t r0, uint32_t r1, Field field, uint8_t* v) {
    int64_t k = 0;
    for (uint32_t r = r0; r < r1; ++r) {
        if (in[r].op != ISL_OP_ALLOC) continue;
        if (k && field(r) != *v) return -1;
        *v = field(r);
        ++k;
    }
    return k;
}

// A canonical GPU range [lo, hi) in storage order (ISL_POLICY_RIGHT_TO_LEFT stores the inventory reversed), or back: its own inverse
std::pair<uint32_t, uint32_t> storage_range(const isl_engine* e, uint32_t lo, uint32_t hi) { return e->prof.flip ? std::make_pair(e->G - hi, e->G - lo) : std::make_pair(lo, hi); }
// Restricts e to canonical ranges (set) for one call, isl_place_batch_range or ISL_FLAG_ALL_NODES; {lo, hi} come back however it returns
struct RangeRestriction {
    isl_engine* e; const uint32_t lo, hi;
    ~RangeRestriction() { e->lo = lo; e->hi = hi; }
    void set(uint32_t a, uint32_t b) { std::tie(e->lo, e->hi) = storage_range(e, a, b); }
};

#define ISL_CUDA(e, call)                                                                    \
    do {                                                                                     \
        cudaError_t _err = (call);                                                           \
        if (_err != cudaSuccess) {                                                           \
            snprintf((e)->cuda_err, sizeof((e)->cuda_err), "%s: %s", #call, cudaGetErrorString(_err)); \
            return ISL_ECUDA;                                                                \
        }                                                                                    \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// What an entry point needs of the engine: the engine states of include/islplace.h, or an open stream (isl_stream_submit / _close).
enum class Needs { nothing, profiles, inventory, ready, open_stream };

// The prologue of every entry point that takes an engine, except the lock-free isl_stream_wait, destroy and the pure getters: the engine
// lock, the state checks, then the engine's device.  rc is ISL_ESTATE while an open stream owns the engine (its resident kernel would keep
// any work enqueued behind the call waiting until isl_stream_close, and the state it runs on must not change under it), or, for the
// stream calls, while none is open; ISL_ESTATE when the tables or the inventory that `needs` names are missing; ISL_ERANGE when a batch of
// n requests exceeds max_batch (Needs::ready).  The state is tested under the lock, so no call can slip in after another thread's
// isl_stream_open.  The device is made current only when rc is ISL_OK; the lock is declared first, so the device is restored before the
// unlock.
struct Entry {
    std::unique_lock<std::mutex> lock;
    std::optional<DeviceGuard> device;
    int rc = ISL_ESTATE;
    Entry(isl_engine* e, Needs needs, uint64_t n = 0) : lock(e->mu) {
        const bool have = needs == Needs::profiles    ? e->have_profiles
                          : needs == Needs::inventory ? e->have_inventory
                          : needs == Needs::ready     ? e->have_profiles && e->have_inventory
                                                      : true;
        if (e->open.active != (needs == Needs::open_stream) || !have) return;
        if (needs == Needs::ready && n > e->cfg.max_batch) { rc = ISL_ERANGE; return; }
        device.emplace(e->device);
        rc = ISL_OK;
    }
};

inline uint32_t ceil_div(uint32_t a, uint32_t b) { return (a + b - 1) / b; }
// SMs a fed stream keeps free for its pre-pass kernels.  On a 132-SM H100 the 128 speculative stages of a 65 536-GPU inventory
// (512 GPUs each), the copier CTA and these three fill the device; a larger reserve leaves such a stream without speculative rounds.
// bench.py config 4 on an H100 SXM (400 W), reserve 3 against 16, two runs each: open stream with one batch in flight 6.8 against
// 26.9 ms per step, with two 5.9-6.1 against 14.1-14.2 ms; the device-resident and per-batch legs and the fed replay unchanged.
// ISL_FEED_RESERVE overrides it for A/B builds (tools/ab_build.sh).
#ifndef ISL_FEED_RESERVE
#define ISL_FEED_RESERVE 3
#endif
constexpr uint32_t kFeedReserve = ISL_FEED_RESERVE;

int check_launch(isl_engine* e, const char* what) {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) { snprintf(e->cuda_err, sizeof(e->cuda_err), "%s: %s", what, cudaGetErrorString(err)); return ISL_ECUDA; }
    ++e->st.kernel_launches;
    return ISL_OK;
}

// One cooperative launch (k_preempt, k_ganglocal): ISL_ECUDA, with the kernel's name, when it does not start.
int launch_cooperative(isl_engine* e, const void* kernel, const char* name, uint32_t grid, uint32_t threads, size_t smem, void** params) {
    const cudaError_t err = cudaLaunchCooperativeKernel(kernel, dim3(grid), dim3(threads), params, smem, e->stream);
    if (err != cudaSuccess) { cudaGetLastError(); snprintf(e->cuda_err, sizeof(e->cuda_err), "%s: %s", name, cudaGetErrorString(err)); return ISL_ECUDA; }
    ++e->st.kernel_launches;
    return ISL_OK;
}

// The nodes [nlo, nhi) that own a GPU of [lo, hi), lo < hi, under the node offsets `off`.
std::pair<uint32_t, uint32_t> node_span(const std::vector<uint32_t>& off, uint32_t lo, uint32_t hi) {
    return {(uint32_t)(std::upper_bound(off.begin(), off.end(), lo) - off.begin()) - 1,
            (uint32_t)(std::upper_bound(off.begin(), off.end(), hi - 1) - off.begin())};
}

// f(std::integral_constant<int, K>) with K = the candidate slots of the loaded tables (k_small<K>, k_chain<K>, k_pipeline<K, ..>)
template <typename F>
auto with_cand_slots(const isl_engine* e, F&& f) {
    switch (e->n_cand_slots) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        default: return f(std::integral_constant<int, 4>{});
    }
}

// The end of a path of one launch, or of k_prepare + one launch (with_prepare): under ISL_FLAG_TIMING ev[0] .. ev[1] are the frees and
// ev[last - 1] .. ev[last] the commit; then the batch counters.
void finish_batch(isl_engine* e, uint32_t n, bool with_prepare) {
    if (e->cfg.flags & ISL_FLAG_TIMING) {
        const uint32_t last = with_prepare ? 2 : 1;
        cudaEventRecord(e->ev[last], e->stream);
        cudaEventSynchronize(e->ev[last]);
        float t;
        if (with_prepare) { cudaEventElapsedTime(&t, e->ev[0], e->ev[1]); e->st.ms_free += t; }
        cudaEventElapsedTime(&t, e->ev[last - 1], e->ev[last]); e->st.ms_commit += t;
        cudaEventElapsedTime(&t, e->ev[0], e->ev[last]); e->st.ms_total += t;
    }
    ++e->st.batches; e->st.requests += n;
}

// The executors of route()'s paths.  Each enqueues only; the caller synchronises.
// k_small: one launch of one CTA resolves a batch, from device memory or inline requests.
int run_small(isl_engine* e, uint32_t n, const uint2* d_in, const SmallReqs* inl, uint2* d_out) {
    static const SmallReqs zero{};
    const SmallReqs& params = inl ? *inl : zero;
    const bool timing = e->cfg.flags & ISL_FLAG_TIMING;
    if (timing) cudaEventRecord(e->ev[0], e->stream);
    with_cand_slots(e, [&](auto k) {
        k_small<decltype(k)::value><<<1, kSmallThreads, 0, e->stream>>>(e->tab, e->prof, n, d_in, params, d_out, e->d_occ, e->d_gtab, e->d_feas, e->G, e->lo,
                                                                         e->hi, e->cand_profiles, e->d_cand, e->d_cand_o16, e->d_ctrl);
    });
    if (int rc = check_launch(e, "k_small")) return rc;
    finish_batch(e, n, false);
    return ISL_OK;
}

// k_few: the shortest path, requests as kernel parameters.
int run_few(isl_engine* e, uint32_t n, const SmallReqs& inl, uint2* d_out) {
    const bool timing = e->cfg.flags & ISL_FLAG_TIMING;
    if (timing) cudaEventRecord(e->ev[0], e->stream);
    k_few<<<1, kFewThreads, 0, e->stream>>>(e->prof, n, inl, d_out, e->d_occ, e->d_gtab, e->d_lut, e->d_sizes, e->n_tables, e->G, e->lo, e->hi, e->d_ctrl);
    if (int rc = check_launch(e, "k_few")) return rc;
    finish_batch(e, n, false);
    return ISL_OK;
}

// k_prepare of one batch in front of a request-major kernel: the frees and the default records, bracketed by ev[0] .. ev[1] under
// ISL_FLAG_TIMING.
int prepare_batch(isl_engine* e, uint32_t n, const uint2* d_in, uint2* d_out) {
    const bool timing = e->cfg.flags & ISL_FLAG_TIMING;
    if (timing) cudaEventRecord(e->ev[0], e->stream);
    k_prepare<<<ceil_div(n, kTile), kTileThreads, 0, e->stream>>>(n, d_in, d_out, reinterpret_cast<uint32_t*>(e->d_occ.get()), e->G, e->lo, e->hi,
                                                                  e->prof, e->d_tile_counts, e->d_ctrl, nullptr, nullptr, 0, 0);
    if (int rc = check_launch(e, "k_prepare")) return rc;
    if (timing) cudaEventRecord(e->ev[1], e->stream);
    return ISL_OK;
}

// What run_bestfit and run_gangs share in front of k_bestfit: the class bitmaps (shared memory up to kBfSmemGpus GPUs of one table, else
// global memory zeroed here), then k_prepare (frees + default records).  *smem = the dynamic shared memory k_bestfit needs.  An empty
// range has no class bitmaps: k_prepare's default records are the whole answer.
int prepare_bestfit(isl_engine* e, uint32_t n, const uint2* d_in, uint2* d_out, size_t* smem) {
    const uint32_t Gr = e->hi - e->lo;
    if (Gr > kBfMaxGpus) return ISL_ERANGE;
    const uint32_t W0 = (Gr + 31) / 32, W1 = (W0 + 31) / 32, stride = W0 + W1;
    const bool in_smem = e->n_tables == 1 && Gr <= kBfSmemGpus;
    *smem = in_smem ? (size_t)256 * stride * sizeof(uint32_t) : 0;
    if (!in_smem && Gr) {   // class bitmaps in global memory: one set of 256 per table, zeroed here (HBM speed) instead of by the lone CTA
        const size_t words = (size_t)256 * e->n_tables * stride;
        ISL_CUDA(e, e->d_bf_bitmaps.reserve(words));
        ISL_CUDA(e, cudaMemsetAsync(e->d_bf_bitmaps, 0, words * sizeof(uint32_t), e->stream));
    }
    return prepare_batch(e, n, d_in, d_out);
}

// ISL_POLICY_BEST_FIT: frees + defaults, then the request-major class-bitmap kernel (one CTA).
int run_bestfit(isl_engine* e, uint32_t n, const uint2* d_in, uint2* d_out) {
    if (n == 0) return ISL_OK;
    size_t smem;
    if (int rc = prepare_bestfit(e, n, d_in, d_out, &smem)) return rc;
    if (e->hi == e->lo) { finish_batch(e, n, true); return ISL_OK; }     // empty range: ALLOCs NO_CAPACITY, every FREE outside it
    // ISL_FLAG_FIRST_AVAILABLE: the pods-of-alternatives loop (a zero score table makes it first-fit, prof.flip right-to-left)
    const bool multi = e->n_tables != 1;
    auto kernel = first_available(e) ? (multi ? k_bestfit<true, false, true> : k_bestfit<false, false, true>) : (multi ? k_bestfit<true> : k_bestfit<false>);
    kernel<<<1, kBfThreads, multi ? 0 : smem, e->stream>>>(n, d_in, d_out, e->d_occ, e->lo, e->hi, e->d_lut, e->prof, e->d_bf_bitmaps, e->d_ctrl, e->d_score,
                                                           e->d_gtab, e->d_sizes, e->n_tables, nullptr, 0);
    if (int rc = check_launch(e, "k_bestfit")) return rc;
    finish_batch(e, n, true);
    return ISL_OK;
}

// ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED: frees + defaults, then k_nodefit (one CTA) over the nodes the range touches.
int run_nodefit(isl_engine* e, uint32_t n, const uint2* d_in, uint2* d_out) {
    if (n == 0) return ISL_OK;
    if (int rc = prepare_batch(e, n, d_in, d_out)) return rc;
    if (e->hi == e->lo) { finish_batch(e, n, true); return ISL_OK; }     // empty range: ALLOCs NO_CAPACITY, every FREE outside it
    uint32_t nlo, nhi;                                          // node scoring stores the inventory in canonical order
    std::tie(nlo, nhi) = node_span(e->node_off, e->lo, e->hi);
    NodeFitArgs a{};
    a.Nr = nhi - nlo;
    for (uint32_t cnt = a.Nr;; cnt = ceil_div(cnt, 32)) {       // level sizes down to the root, each padded to 32 keys
        a.lvl_off[a.levels] = a.T; a.lvl_cnt[a.levels++] = cnt;
        a.T += (cnt + 31u) & ~31u;
        if (cnt == 1) break;
    }
    auto& nf = e->nf;
    const bool in_smem = a.Nr <= kNfSmemNodes;
    ISL_CUDA(e, nf.fit.reserve((size_t)e->prof.n * a.Nr));
    ISL_CUDA(e, nf.nodes.reserve((size_t)2 * a.Nr));
    if (!in_smem) ISL_CUDA(e, nf.tree.reserve((size_t)e->prof.n * a.T));
    a.in = d_in; a.out = d_out; a.occ = e->d_occ; a.gtab = e->d_gtab; a.lut = e->d_lut; a.sizes = e->d_sizes; a.node_off = nf.node_off;
    a.tree = nf.tree; a.fit = nf.fit; a.busy = nf.nodes; a.meta = nf.nodes + a.Nr; a.ctrl = e->d_ctrl;
    a.n = n; a.lo = e->lo; a.hi = e->hi; a.nlo = nlo; a.most = e->cfg.policy == ISL_POLICY_MOST_ALLOCATED;
    memcpy(a.width, nf.width, sizeof a.width);
    (first_available(e) ? k_nodefit<true> : k_nodefit<false>)<<<1, kNfThreads, in_smem ? (size_t)e->prof.n * a.T * sizeof(uint32_t) : 0, e->stream>>>(a, e->prof.n);
    if (int rc = check_launch(e, "k_nodefit")) return rc;
    finish_batch(e, n, true);
    return ISL_OK;
}

// isl_place_gangs, every policy: frees + defaults, then k_bestfit's gang instantiation over the n_gangs + 1 offsets at d_gang_off.
int run_gangs(isl_engine* e, uint32_t n_gangs, const uint32_t* d_gang_off, uint32_t n, const uint2* d_in, uint2* d_out) {
    size_t smem;
    if (int rc = prepare_bestfit(e, n, d_in, d_out, &smem)) return rc;
    if (e->n_tables == 1)
        k_bestfit<false, true><<<1, kBfThreads, smem, e->stream>>>(n, d_in, d_out, e->d_occ, e->lo, e->hi, e->d_lut, e->prof, e->d_bf_bitmaps, e->d_ctrl, e->d_score,
                                                                   e->d_gtab, e->d_sizes, 1, d_gang_off, n_gangs);
    else
        k_bestfit<true, true><<<1, kBfThreads, 0, e->stream>>>(n, d_in, d_out, e->d_occ, e->lo, e->hi, e->d_lut, e->prof, e->d_bf_bitmaps, e->d_ctrl, e->d_score,
                                                               e->d_gtab, e->d_sizes, e->n_tables, d_gang_off, n_gangs);
    if (int rc = check_launch(e, "k_bestfit (gangs)")) return rc;
    finish_batch(e, n, true);
    return ISL_OK;
}

// The layout of k_ganglocal and k_preempt_gangs, over the nodes the partition touches: each CTA gets whole nodes, about Gr / grid GPUs
// (one CTA per SM at most, one per 512 GPUs below that, never more than nodes), and `per_gpu` bytes per GPU of its share (rounded up to 16
// GPUs) in shared memory when they fit in `smem_optin` (the kernel's dynamic shared memory opt-in), else *smem_out = 0 and the caller
// keeps them in global memory (a.scratch).  Fills every other field of `a`, a.share in GPUs; *nodes = the nodes the partition touches.
int gang_layout(isl_engine* e, const void* kernel, int smem_optin, uint32_t per_gpu, uint32_t n_gangs, const uint32_t* d_gang_off,
                const uint2* d_in, uint2* d_out, GangNodeArgs& a, uint32_t* grid_out, size_t* smem_out, uint32_t* nodes) {
    auto& gn = e->gn;
    const uint32_t Gr = e->hi - e->lo;
    uint32_t nlo, nhi;
    std::tie(nlo, nhi) = node_span(gn.off, e->lo, e->hi);
    int sms = 0, per_sm = 0;
    ISL_CUDA(e, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device));
    const uint32_t grid = std::max(1u, std::min({(uint32_t)sms, kGnMaxCtas, ceil_div(Gr, 512), nhi - nlo}));
    a = GangNodeArgs{};
    uint32_t share = 0;                                     // the largest share, in GPUs
    auto local = [&](uint32_t j) { return std::min(std::max(gn.off[nlo + j], e->lo), e->hi) - e->lo; };
    for (uint32_t c = 1; c <= grid; ++c) {
        const uint32_t target = e->lo + (uint32_t)((uint64_t)Gr * c / grid);
        a.cta_node[c] = c == grid ? nhi - nlo : (uint32_t)(std::lower_bound(gn.off.begin() + nlo, gn.off.begin() + nhi, target) - gn.off.begin()) - nlo;
        share = std::max(share, local(a.cta_node[c]) - local(a.cta_node[c - 1]));
    }
    // the bytes of a share in shared memory when they fit, else in global memory
    size_t smem = ((size_t)share + 15) / 16 * 16 * per_gpu;
    if (smem > (size_t)smem_optin ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kGnThreads, smem) != cudaSuccess || per_sm < 1) {
        cudaGetLastError();
        smem = 0;
    }
    ISL_CUDA(e, gn.keys.reserve((size_t)2 * grid));
    a.in = d_in; a.out = d_out; a.occ = e->d_occ; a.gtab = e->d_gtab; a.lut = e->d_lut; a.score = e->d_score; a.sizes = e->d_sizes;
    a.node_off = gn.node_off; a.gang_off = d_gang_off; a.keys = gn.keys; a.ctrl = e->d_ctrl;
    a.n_gangs = n_gangs; a.n_tables = e->n_tables; a.lo = e->lo; a.hi = e->hi; a.nlo = nlo; a.share = (uint32_t)(smem / per_gpu);
    *grid_out = grid; *smem_out = smem; *nodes = nhi - nlo;
    return ISL_OK;
}

// isl_place_gangs on an engine with a k_ganglocal instantiation (gang.place): frees + defaults, then one cooperative launch of it
// (gang_layout with its opt-in).  An instantiation of kLocPerGang places each gang by the byte at d_locality[gang], and one of kMin
// reads each gang's minimum m' from the uint32 words that follow the bytes (rounded up to 4).  CTA c of an instantiation that runs
// distinct-node gangs stacks its wins in gn.wins[cta_node[c] ..), at most one per node it owns; a balanced instantiation keeps the
// count of node j in gn.wins[j] as well.
int run_ganglocal(isl_engine* e, uint32_t n_gangs, const uint32_t* d_gang_off, const uint8_t* d_locality, uint32_t n,
                  const uint2* d_in, uint2* d_out) {
    const GangKernel& k = *e->gang.place;
    if (int rc = prepare_batch(e, n, d_in, d_out)) return rc;
    GangScoreArgs a;            // the node-scored instantiations read all of it, the others its GangNodeArgs part
    uint32_t grid, nodes;
    size_t smem;
    if (int rc = gang_layout(e, k.fn, e->gn.optin, 2, n_gangs, d_gang_off, d_in, d_out, a, &grid, &smem, &nodes)) return rc;
    memcpy(a.width, e->nf.width, sizeof a.width);
    a.most = e->cfg.policy == ISL_POLICY_MOST_ALLOCATED;
    if (!smem) ISL_CUDA(e, e->gn.scratch.reserve(e->hi - e->lo));     // the second byte per GPU; the live bytes are the occupancy
    a.scratch = e->gn.scratch;
    if (k.loc == ISL_GANG_DISTINCT_NODES || k.loc == kLocPerGang) ISL_CUDA(e, e->gn.wins.reserve(nodes));
    uint2* wins = e->gn.wins;
    void* params[] = {&a, &e->prof, &wins, &d_locality};
    if (int rc = launch_cooperative(e, k.fn, k.name, grid, kGnThreads, smem, params)) return rc;
    finish_batch(e, n, true);
    return ISL_OK;
}

// The chunk path: k_prepare, then per chunk of kChunk requests k_partition, the two sweeps, k_chain and k_commit.  d_heads_in / d_heads_out
// (isl_place_batch_partitioned): the queue-head token per chunk, carried by the caller from the engine of the previous GPU range.
int run_chunks(isl_engine* e, uint32_t n, const uint2* d_in, uint2* d_out, const uint32_t* d_heads_in, uint32_t* d_heads_out) {
    if (n == 0) return ISL_OK;
    const bool timing = e->cfg.flags & ISL_FLAG_TIMING;
    const uint32_t tiles = ceil_div(n, kTile);
    if (timing) cudaEventRecord(e->ev[0], e->stream);
    k_prepare<<<tiles, kTileThreads, 0, e->stream>>>(n, d_in, d_out, reinterpret_cast<uint32_t*>(e->d_occ.get()), e->G, e->lo, e->hi,
                                                     e->prof, e->d_tile_counts, e->d_ctrl, nullptr, nullptr, 0, 0);
    if (int rc = check_launch(e, "k_prepare")) return rc;
    if (timing) cudaEventRecord(e->ev[1], e->stream);
    const uint32_t first_block = e->lo / kSweepBlock;
    const uint32_t sweep_blocks = e->hi > e->lo ? ceil_div(e->hi, kSweepBlock) - first_block : 0;
    float ms_part = 0, ms_sweep = 0, ms_commit = 0;
    for (uint32_t c0 = 0; c0 < n; c0 += kChunk) {
        const uint32_t n_chunk = std::min(kChunk, n - c0);
        const uint32_t first_tile = c0 / kTile, n_tiles = ceil_div(n_chunk, kTile);
        if (timing) cudaEventRecord(e->ev[2], e->stream);
        k_partition<<<n_tiles, kTileThreads, 0, e->stream>>>(n_chunk, d_in + c0, e->prof.n, e->d_tile_counts + (size_t)first_tile * ISL_MAX_PROFILES,
                                                             n_tiles, e->cand_profiles, e->d_q, e->d_ctrl, nullptr, 0, 0);
        if (int rc = check_launch(e, "k_partition")) return rc;
        if (timing) cudaEventRecord(e->ev[3], e->stream);
        const uint32_t* h_in = d_heads_in ? d_heads_in + (size_t)(c0 / kChunk) * ISL_MAX_PROFILES : nullptr;
        uint32_t* h_out = d_heads_out ? d_heads_out + (size_t)(c0 / kChunk) * ISL_MAX_PROFILES : nullptr;
        if (h_out) {
            if (h_in) ISL_CUDA(e, cudaMemcpyAsync(h_out, h_in, ISL_MAX_PROFILES * sizeof(uint32_t), cudaMemcpyDeviceToDevice, e->stream));
            else ISL_CUDA(e, cudaMemsetAsync(h_out, 0, ISL_MAX_PROFILES * sizeof(uint32_t), e->stream));
        }
        if (sweep_blocks) {     // candidate compaction — or, for a single-profile chunk, the capacity scan that commits directly
            k_sweep_count<<<sweep_blocks, kSweepThreads, 0, e->stream>>>(reinterpret_cast<const uint4*>(e->d_occ.get()), reinterpret_cast<const uint4*>(e->d_gtab.get()), e->d_feas, first_block, e->lo, e->hi,
                                                                         e->d_ctrl, e->d_sweep_counts, e->d_capn);
            if (int rc = check_launch(e, "k_sweep_count")) return rc;
            k_sweep_scatter<<<sweep_blocks, kSweepThreads, 0, e->stream>>>(reinterpret_cast<const uint4*>(e->d_occ.get()), reinterpret_cast<const uint4*>(e->d_gtab.get()), e->d_feas, first_block, e->lo, e->hi,
                                                                           e->d_ctrl, e->d_sweep_counts, e->d_cand, e->d_cand_o16, e->d_capn, e->d_seq, e->d_q, e->d_occ,
                                                                           d_out + c0, h_in, h_out, e->d_sizes, e->prof.flip);
            if (int rc = check_launch(e, "k_sweep_scatter")) return rc;
        }
        if (timing) cudaEventRecord(e->ev[4], e->stream);
        with_cand_slots(e, [&](auto k) {      // dynamic shared memory opted in per device by isl_create
            k_chain<decltype(k)::value><<<1, kChainThreads, (size_t)kQCap * sizeof(uint16_t), e->stream>>>(e->tab, e->d_ctrl, e->d_q, e->d_cand_o16, e->d_feas,
                                                                                                    e->d_log, h_in, h_out);
        });
        if (int rc = check_launch(e, "k_chain")) return rc;
        k_commit<<<kChunk / 256, 256, 0, e->stream>>>(e->d_ctrl, e->d_log, e->d_cand, reinterpret_cast<uint32_t*>(e->d_occ.get()), d_out + c0, e->prof.flip);
        if (int rc = check_launch(e, "k_commit")) return rc;
        if (timing) {
            cudaEventRecord(e->ev[5], e->stream);
            cudaEventSynchronize(e->ev[5]);
            float t;
            cudaEventElapsedTime(&t, e->ev[2], e->ev[3]); ms_part += t;
            cudaEventElapsedTime(&t, e->ev[3], e->ev[4]); ms_sweep += t;
            cudaEventElapsedTime(&t, e->ev[4], e->ev[5]); ms_commit += t;
        }
    }
    if (timing) {
        float t;
        cudaEventElapsedTime(&t, e->ev[0], e->ev[1]); e->st.ms_free += t;     // prepare = frees + defaults + histogram
        e->st.ms_partition += ms_part; e->st.ms_sweep += ms_sweep; e->st.ms_commit += ms_commit;
        cudaEventElapsedTime(&t, e->ev[0], e->ev[5]); e->st.ms_total += t;
    }
    ++e->st.batches;
    e->st.requests += n;
    return ISL_OK;
}


// One cooperative launch of k_pipeline<K, P15, Spec> for the loaded tables.  P15: profile index 15 is in use, the pop test needs the
// slower, INF-safe form.
int start_pipeline(isl_engine* e, PipeArgs& args) {
    const bool p15 = e->prof.n == ISL_MAX_PROFILES;
    void* kernel = with_cand_slots(e, [&](auto k) {
        constexpr int K = decltype(k)::value;
        return p15 ? (args.spec ? (void*)k_pipeline<K, true, true> : (void*)k_pipeline<K, true, false>)
                   : (args.spec ? (void*)k_pipeline<K, false, true> : (void*)k_pipeline<K, false, false>);
    });
    void* params[] = {&e->tab, &args};
    const cudaError_t err = cudaLaunchCooperativeKernel(kernel, dim3(args.n_seg + (args.copier ? 1u : 0u)), dim3(kPipeThreads), params, kPipeSmem, e->stream);
    if (err == cudaErrorCooperativeLaunchTooLarge || err == cudaErrorLaunchOutOfResources) {   // e.g. the GPU is shared: not all CTAs can be co-resident
        cudaGetLastError();
        return ISL_ESTATE;          // caller falls back to the chunk-by-chunk path
    }
    if (err != cudaSuccess) { snprintf(e->cuda_err, sizeof(e->cuda_err), "cudaLaunchCooperativeKernel: %s", cudaGetErrorString(err)); return ISL_ECUDA; }
    ++e->st.kernel_launches;
    return ISL_OK;
}

int query_coresident(isl_engine* e) {
    if (e->max_coresident) return ISL_OK;
    int per_sm = 0, sms = 0, coop = 0;
    ISL_CUDA(e, cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, e->device));
    ISL_CUDA(e, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device));
    ISL_CUDA(e, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pipeline<4, true, true>, kPipeThreads, kPipeSmem));
    e->max_coresident = coop ? std::max(1, per_sm * sms) : -1;
    return ISL_OK;
}

// Segment geometry of the pipeline for a stream of n_chunks chunks of ~avg_chunk requests; seg_cap: the largest segment whose queue
// windows fit in shared memory.  ISL_ERANGE: the inventory does not fit the co-resident CTAs (or the tables need too many candidates per
// segment).
int segment_geometry(isl_engine* e, uint32_t n_chunks, double avg_chunk, bool want_feed, uint32_t seg_cap, bool spec, PipePlan* p) {
    if (int rc = query_coresident(e)) return rc;
    const uint32_t range = e->hi - e->lo;
    // Segments aimed for.  A batch's decisions form ONE sequential chain over the inventory, only different chunks overlap, so a
    // stream of B chunks over S stages takes about (S + B - 1) x (D x t_dec / S + t_fix), D = decisions of a chunk.  tools/chain_cost.py
    // on config 4, H100 80GB HBM3 (SXM, 700 W power limit, SM clock 1980 MHz): t_dec = 32.6 ns per decision, t_fix = 1.57 us per busy
    // cell (token in -> loop start 1.45 us, loop end -> token out 0.12 us; profiles/r03_chain_sm90.md).  Minimum at
    // S = sqrt((B - 1) x D x t_dec / t_fix); D is estimated by the smaller of the chunk size and ~3.5 placements per GPU.
    // ISL_PIPE_SEGMENTS overrides (experiments).
    constexpr double kTdecUs = 0.0326, kTfixUs = 1.57;
    const uint32_t stages_max = (uint32_t)std::max(1, e->max_coresident);     // one CTA per SM: the SM count of the device
    uint32_t target = stages_max;
    {
        const double d_est = std::min(avg_chunk, 3.5 * (double)e->G);
        const double s_opt = std::sqrt(std::max(1.0, (double)n_chunks - 1.0) * d_est * (kTdecUs / kTfixUs));
        target = (uint32_t)std::min((double)stages_max, std::max(1.0, std::floor(s_opt + 0.5)));
    }
    if (spec) target = stages_max;      // speculative rounds: every stage works in every round — as many (short) segments as there are SMs
    if (const char* v = getenv("ISL_PIPE_SEGMENTS")) target = std::max(1u, (uint32_t)strtoul(v, nullptr, 10));
    target = std::min(target, (uint32_t)std::max(1, e->max_coresident));
    // fed host streams run their per-batch pre-pass kernels WHILE the pipeline is resident: keep kFeedReserve SMs free of pipeline
    // CTAs (one CTA fills an SM's shared memory, and kernels with another shared-memory carve-out cannot join it there)
    if (want_feed && e->max_coresident > 2 * (int)kFeedReserve) target = std::min(target, (uint32_t)e->max_coresident - 1u - kFeedReserve);
    // segment size from the WHOLE inventory: a partitioned rank keeps the global pipeline depth (~target stages over all ranks)
    if (seg_cap < 64 || e->max_coresident <= 0) return ISL_ERANGE;
    // one sweep / chain / commit round covers `sub` GPUs; an inventory beyond target x sub gives every stage several sub-segments
    const uint32_t sub = std::min(seg_cap, std::max(64u, (ceil_div(e->G, target) + 63u) / 64u * 64u));
    // a short stream wants few stages, a large inventory needs many (a stage holds at most kSubMax sub-segments): the inventory wins
    const uint32_t stages_avail = (want_feed && e->max_coresident > 2 * (int)kFeedReserve) ? (uint32_t)e->max_coresident - 1u - kFeedReserve : (uint32_t)e->max_coresident;
    target = std::max(target, std::min(stages_avail, ceil_div(ceil_div(e->G, sub), kSubMax)));
    const uint32_t n_sub = std::max(1u, ceil_div(ceil_div(e->G, sub), target));
    if (n_sub > kSubMax) return ISL_ERANGE;
    const uint32_t seg = sub * n_sub;
    const uint32_t n_seg = std::max(1u, ceil_div(range, seg));
    if (n_seg > (uint32_t)e->max_coresident) return ISL_ERANGE;
    p->seg = seg; p->n_seg = n_seg; p->sub = sub;
    return ISL_OK;
}

// The pipeline of one call over n_chunks chunks of ~avg_chunk requests, with or without speculative rounds (isl_kernels.cuh,
// DESIGN.md 4.5).  The mode is e->spec_mode, or ISL_SPEC=0|1 from the environment; auto_spec: what ISL_SPEC_AUTO means for the caller;
// spec_allowed: the caller's own limits permit speculation; spec_feed_room: a speculative plan must also leave the copier CTA and the
// feed reserve free.  Speculative rounds need one sub-segment per stage; a plan without them is the fallback.  ISL_ERANGE: see
// segment_geometry — the caller takes the chunk-by-chunk path.
int plan_pipeline(isl_engine* e, uint32_t n_chunks, double avg_chunk, bool want_feed, bool ring, bool auto_spec, bool spec_allowed,
                  bool spec_feed_room, PipePlan* p) {
    uint32_t total_cand = 0;
    for (uint32_t k = 0; k < 4; ++k) for (uint32_t l = 0; l < 32; ++l) total_cand += e->tab.desc[k][l] >> 31;
    const uint32_t seg_cap = max_segment_for(total_cand);      // queue windows of a segment must fit in shared memory
    uint32_t mode = e->spec_mode;
    if (const char* v = getenv("ISL_SPEC")) mode = atoi(v) ? ISL_SPEC_ON : ISL_SPEC_OFF;
    *p = PipePlan{};
    if (spec_allowed && !(ring && e->spec_world < 2) && kPipeThreads >= 208 && (mode == ISL_SPEC_ON || (mode == ISL_SPEC_AUTO && auto_spec))) {
        const uint32_t range = e->hi - e->lo;
        if (ring) {
            // one sequence of stages over all ranks: a power-of-two stage size that every rank boundary is a multiple of (all ranks evaluate
            // the same predicate over the same bounds, so they agree)
            uint32_t sz = 64;
            while (ceil_div(e->G, sz) > kSpecMaxStages) sz *= 2;
            bool ok = sz <= kSegMax && e->spec_world == e->ring_world && n_chunks <= e->d_spec.cap() && e->spec_bounds[e->spec_world] == e->G &&
                      e->spec_bounds[e->spec_rank] == e->lo && e->spec_bounds[e->spec_rank + 1] == e->hi && query_coresident(e) == ISL_OK;
            for (uint32_t r = 0; ok && r <= e->spec_world; ++r) ok = e->spec_bounds[r] % sz == 0 || e->spec_bounds[r] == e->G;
            for (uint32_t r = 0; ok && r < e->spec_world; ++r) ok = e->spec_bounds[r] < e->spec_bounds[r + 1] && ceil_div(e->spec_bounds[r + 1] - e->spec_bounds[r], sz) <= (uint32_t)std::max(1, e->max_coresident);
            if (ok && sz <= seg_cap) { p->seg = p->sub = sz; p->n_seg = ceil_div(range, sz); p->spec = true; return ISL_OK; }
        } else {
            const int rc = segment_geometry(e, n_chunks, avg_chunk, want_feed, seg_cap, true, p);
            if (rc == ISL_ECUDA) return rc;
            p->spec = rc == ISL_OK && p->seg == p->sub && p->n_seg <= kSpecMaxStages && p->n_seg >= 2 &&
                      (!spec_feed_room || p->n_seg + 1 + kFeedReserve <= (uint32_t)e->max_coresident);
            if (p->spec) return ISL_OK;
        }
    }
    return segment_geometry(e, n_chunks, avg_chunk, want_feed, seg_cap, false, p);
}

constexpr unsigned long long kOpenWaitNs = 600000000000ull;     // open streams may idle between batches: 10 min

// record memory for n_chunks chunks; the words carry the call epoch (24 bits) — cleared when (re)allocated and when those bits wrap
int prepare_spec(isl_engine* e, uint32_t n_chunks, uint32_t epoch, cudaStream_t st) {
    if (e->spec_shared) return n_chunks <= e->d_spec.cap() ? ISL_OK : ISL_ERANGE;      // peers hold a mapping of it: fixed size, tags carry the stream id
    bool fresh;
    ISL_CUDA(e, e->d_spec.reserve(n_chunks, Growth::headroom, &fresh));
    const bool wrapped = (epoch >> 24) != e->spec_hi;
    if (fresh || wrapped) ISL_CUDA(e, cudaMemsetAsync(e->d_spec, 0, e->d_spec.bytes(), st));
    e->spec_hi = epoch >> 24;
    return ISL_OK;
}

// A tool that serialises kernels is around: ncu and compute-sanitizer inject through the first variable, CUDA_LAUNCH_BLOCKING is the
// second.  A pipeline that waits for kernels launched after it would starve.
bool kernels_serialised() {
    return getenv("CUDA_INJECTION64_PATH") || getenv("CUDA_LAUNCH_BLOCKING") || getenv("NV_COMPUTE_PROFILER_PERFWORKS_DIR");
}

int ensure_feed_stream(isl_engine* e) {
    if (e->feed_stream) return ISL_OK;
    ISL_CUDA(e, cudaStreamCreateWithFlags(e->feed_stream.out(), cudaStreamNonBlocking));
    ISL_CUDA(e, cudaEventCreateWithFlags(e->ev_feed.out(), cudaEventDisableTiming));
    ISL_CUDA(e, cudaEventCreateWithFlags(e->ev_feed_done.out(), cudaEventDisableTiming));
    return ISL_OK;
}

// The epoch of a new pipeline launch.
int next_epoch(isl_engine* e, uint32_t* epoch) {
    *epoch = ++e->epoch;
    if ((*epoch & 0x7FFFu) == 0) *epoch = ++e->epoch;      // the token words carry the low 15 bits as a tag; tag 0 is what a cleared buffer holds
    if ((*epoch & 0x7FFFu) == 1 && *epoch != 1 && e->d_tokens)    // tag wrap-around: no stale word of 32 768 calls ago may look current
        ISL_CUDA(e, cudaMemsetAsync(e->d_tokens, 0, e->d_tokens.bytes(), e->stream));
    return ISL_OK;
}

// Device tables of a pipeline over n_chunks chunks (queues of q_stride entries, n_seg + 1 tokens each), n_tiles pre-pass tiles and the
// free masks of n_batches batches; n_ready ready flags and n_done done counters (0: none needed).
int grow_stream_buffers(isl_engine* e, uint32_t n_chunks, uint32_t q_stride, uint32_t n_tiles, uint32_t n_batches, uint32_t n_seg,
                        uint32_t n_ready, uint32_t n_done) {
    ISL_CUDA(e, e->d_chunks.reserve(n_chunks, Growth::headroom));
    ISL_CUDA(e, e->d_cctl.reserve(n_chunks, Growth::headroom));
    ISL_CUDA(e, e->d_qall.reserve((size_t)n_chunks * q_stride, Growth::headroom));
    ISL_CUDA(e, e->d_tiles.reserve(n_tiles, Growth::headroom));
    ISL_CUDA(e, e->d_free_acc.reserve((size_t)n_batches * (e->occ_bytes / 4), Growth::headroom));
    bool fresh;     // token flags carry the call epoch: a (re)allocated buffer must not hold stale flags of an earlier owner
    ISL_CUDA(e, e->d_tokens.reserve((size_t)n_chunks * (n_seg + 1), Growth::headroom, &fresh));
    if (fresh) ISL_CUDA(e, cudaMemsetAsync(e->d_tokens, 0, e->d_tokens.bytes(), e->stream));
    ISL_CUDA(e, e->d_ready.reserve(n_ready, Growth::headroom));
    ISL_CUDA(e, e->d_done_cnt.reserve(n_done, Growth::headroom));
    return ISL_OK;
}

// Descriptors of batch b, requests [off, off + n) of the stream: pipeline chunks of pc requests (the FREEs of a batch belong to its first
// chunk) and tiles of kTile requests for the two pre-pass launches, stored at chunks[n_chunks] and tiles[n_tiles] on; both counts advance.
void describe_batch(uint32_t b, uint32_t off, uint32_t n, uint32_t pc, ChunkDesc* chunks, uint32_t& n_chunks, TileDesc* tiles, uint32_t& n_tiles) {
    const uint32_t batch_first_tile = n_tiles;
    for (uint32_t c0 = 0; c0 < n; c0 += pc) {
        const uint32_t cn = std::min(pc, n - c0), chunk = n_chunks++;
        const uint32_t chunk_first_tile = n_tiles, chunk_tiles = ceil_div(cn, kTile);
        chunks[chunk] = ChunkDesc{off + c0, cn, b, c0 == 0 ? 1u : 0u};
        for (uint32_t t = 0; t < chunk_tiles; ++t)
            tiles[n_tiles++] = TileDesc{off, n, b, batch_first_tile, chunk, chunk_first_tile, chunk_tiles, off + c0, cn, 0, 0, 0};
    }
}

// The PipeArgs fields every k_pipeline launch shares; the callers add feeding, delivery, windows, rings and tracing.
PipeArgs pipe_args(const isl_engine* e, const PipePlan& plan, uint32_t n_chunks, uint32_t epoch, uint32_t q_stride, uint2* out) {
    PipeArgs args{};
    args.n_chunks = n_chunks; args.n_seg = plan.n_seg; args.seg = plan.seg; args.sub = plan.sub; args.lo = e->lo; args.hi = e->hi; args.epoch = epoch;
    args.flip = e->prof.flip; args.wait_ns = e->wait_ns;
    args.chunks = e->d_chunks; args.cctl = e->d_cctl; args.q_all = e->d_qall; args.free_acc = reinterpret_cast<const uint8_t*>(e->d_free_acc.get());
    args.q_stride = q_stride; args.free_stride = (uint32_t)e->occ_bytes; args.tokens = e->d_tokens; args.occ = e->d_occ; args.gtab = e->d_gtab;
    args.out = out; args.feas = e->d_feas; args.stats = e->d_ctrl;
    if (plan.spec) { args.spec = 1; args.spec_mem = e->d_spec; args.spec_total = plan.n_seg; }
    return args;
}

// A placement call: n_batches batches, resolved one after the other.  Host calls stage through d_req / d_res and end with the results in
// the caller's host buffer; src inline_host: <= kSmallInline host records, which can travel as kernel parameters.
enum class Src { inline_host, host, device };
struct Call {
    uint32_t n_batches; const uint32_t* sizes;
    Src src; const void* in; void* out;     // host or device memory, as src says
    uint32_t xepoch = 0;                    // stream id of a partitioned inventory (isl_place_stream_partitioned; 0: none)
    bool mixed = false;                     // one host batch of >= 4096 requests that mixes placeable profiles
};

enum class Path { few, small, chunks, bestfit, nodefit, pipeline };
struct Route {
    Path path = Path::chunks;
    PipePlan plan; bool feed = false; uint32_t window = 0;      // Path::pipeline: its plan, feed mode, causal window
};

// Which path a call of total (> 0) requests in n_chunks pipeline chunks takes (DESIGN.md 4.3), into a default Route.  Launches nothing.
// ISL_ERANGE: a ring that cannot run as one pipeline; ISL_ECUDA: the co-residency query failed.
int route(isl_engine* e, const Call& c, uint64_t total, uint32_t n_chunks, Route* r) {
    const uint32_t flags = e->cfg.flags, range = e->hi - e->lo, n = c.sizes[0];
    const bool ring = c.xepoch != 0;        // partitioned inventory: tokens cross ranks through peer memory, pipeline mandatory
    if (ring && n_chunks > kMaxStreamChunks) return ISL_ERANGE;
    // latency paths: one batch of <= kSmallMax requests in one CTA (k_small); <= kFewMax inline requests on <= kFewGpus GPUs (k_few)
    if (c.n_batches == 1 && !ring && n <= kSmallMax && !request_major(e->cfg) && !(flags & (ISL_FLAG_NO_SMALL | ISL_FLAG_FORCE_PIPELINE)) &&
        range > 0 && range <= (1u << 18)) {
        const bool few = c.src == Src::inline_host && n <= kFewMax && e->hi - (e->lo & ~15u) <= kFewGpus && !getenv("ISL_NO_FEW");
        r->path = few ? Path::few : Path::small;
        return ISL_OK;
    }
    if (request_major(e->cfg)) { r->path = node_scoring(e->cfg.policy) ? Path::nodefit : Path::bestfit; return ISL_OK; }
    const bool pipeline = ring || (!(flags & ISL_FLAG_NO_PIPELINE) && range > 0 && (n_chunks >= 2 || c.mixed || (flags & ISL_FLAG_FORCE_PIPELINE)));
    if (!pipeline) return ISL_OK;
    // the pipeline keeps one free-mask byte per GPU and batch: very long streams over large inventories go batch by batch
    if ((uint64_t)c.n_batches * e->occ_bytes > (256ull << 20)) return ring ? ISL_ERANGE : ISL_OK;
    // feed mode: host buffers, >= 2 batches, no phase timing / tracing, no kernel-serialising tool around, no ISL_NO_FEED=1 (by hand)
    const bool want_feed = c.src == Src::host && c.n_batches >= 2 && !(flags & (ISL_FLAG_TIMING | ISL_FLAG_TRACE)) && !ring && !getenv("ISL_NO_FEED") &&
                           !kernels_serialised();
    r->window = (ring && e->ring_world == 0) ? 0u : e->window;      // a ring counts the ranks of a window on the owner
    const bool auto_spec = c.n_batches == 1 || (r->window >= 1 && r->window <= 3);        // speculative rounds by default
    // Record words of the rounds carry 24 bits of their call's tag, and shared record memory (isl_ipc_spec_handle) is cleared only when
    // it is allocated: a ring speculates only under a stream id below 2^24, so that no two calls share a tag (every rank sees the same
    // id and takes the same path), and an engine whose record memory is shared speculates on the ring only, where the stream id tags
    // the words, never on calls tagged with its own epoch.
    const bool spec_allowed = ring ? c.xepoch < kSpecRingIds : !e->spec_shared;
    const int rc = plan_pipeline(e, n_chunks, (double)total / n_chunks, want_feed, ring, auto_spec, spec_allowed, false, &r->plan);
    if (rc == ISL_ECUDA) return rc;
    if (rc) return ring ? ISL_ERANGE : ISL_OK;
    r->path = Path::pipeline;
    // feeding also needs room for the copier CTA plus the reserve: the pre-pass could starve behind a full house of pipeline CTAs
    r->feed = want_feed && r->plan.n_seg + 1 + kFeedReserve <= (uint32_t)e->max_coresident;
    return ISL_OK;
}

// Path::chunks / Path::bestfit / Path::nodefit: one batch after the other
int run_batches(isl_engine* e, const Call& c, const uint2* d_in, uint2* d_out, Path path) {
    uint64_t off = 0;
    for (uint32_t b = 0; b < c.n_batches; off += c.sizes[b++])
        if (int rc = path == Path::bestfit   ? run_bestfit(e, c.sizes[b], d_in + off, d_out + off)
                     : path == Path::nodefit ? run_nodefit(e, c.sizes[b], d_in + off, d_out + off)
                                             : run_chunks(e, c.sizes[b], d_in + off, d_out + off, nullptr, nullptr)) return rc;
    return ISL_OK;
}

// Path::pipeline: the pre-pass of every batch, then ONE cooperative k_pipeline.  With r.feed the batches are copied and pre-passed one by
// one on the feed stream while the pipeline runs (it waits per batch on a device flag), and an extra CTA copies every finished chunk's
// results into the caller's buffer when that is mapped pinned memory (*delivered).  A refused launch falls back to the chunk path.
int run_pipeline(isl_engine* e, const Call& c, const Route& r, const uint2* d_in, uint2* d_out, uint64_t total, uint32_t n_chunks, bool* delivered) {
    const uint32_t pc = e->pipe_chunk, n_batches = c.n_batches, *sizes = c.sizes, xepoch = c.xepoch, window = r.window;
    const uint2* h_in = static_cast<const uint2*>(c.in);          // feed: the caller's host buffer
    const PipePlan& plan = r.plan;
    const bool ring = xepoch != 0, feed = r.feed, timing = e->cfg.flags & ISL_FLAG_TIMING;
    uint32_t n_tiles_total = 0;         // pipe_chunk is a whole number of tiles: no tile spans two chunks
    for (uint32_t b = 0; b < n_batches; ++b) n_tiles_total += ceil_div(sizes[b], kTile);
    e->h_chunks.resize(n_chunks); e->h_tiles.resize(n_tiles_total);
    for (uint32_t b = 0, off = 0, chunk = 0, tile = 0; b < n_batches; off += sizes[b++])
        describe_batch(b, off, sizes[b], pc, e->h_chunks.data(), chunk, e->h_tiles.data(), tile);
    const uint32_t q_stride = pc + kQPad * ISL_MAX_PROFILES, free_stride = (uint32_t)e->occ_bytes;      // free_stride: bytes per batch
    const bool need_done = feed || window;
    if (int rc = grow_stream_buffers(e, n_chunks, q_stride, n_tiles_total, n_batches, plan.n_seg, feed ? n_batches + 1 : 0, need_done ? n_chunks : 0)) return rc;
    if (n_tiles_total > ceil_div(e->cfg.max_batch, kTile) + 4096) return ISL_ERANGE;
    uint2* h_out_dev = nullptr;
    if (feed) {     // the feed stream starts behind whatever the engine's stream still holds (earlier calls, load_inventory)
        cudaPointerAttributes pa{};
        if (cudaPointerGetAttributes(&pa, c.out) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer) h_out_dev = static_cast<uint2*>(pa.devicePointer);
        cudaGetLastError();
        if (int rc = ensure_feed_stream(e)) return rc;
        ISL_CUDA(e, cudaEventRecord(e->ev_feed, e->stream));
        ISL_CUDA(e, cudaStreamWaitEvent(e->feed_stream, e->ev_feed, 0));
    }
    const cudaStream_t pre = feed ? e->feed_stream : e->stream;     // the stream the tables and the pre-pass go to
    if (need_done) ISL_CUDA(e, cudaMemsetAsync(e->d_done_cnt, 0, (size_t)n_chunks * sizeof(uint32_t), pre));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_chunks, e->h_chunks.data(), n_chunks * sizeof(ChunkDesc), cudaMemcpyHostToDevice, pre));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_tiles, e->h_tiles.data(), n_tiles_total * sizeof(TileDesc), cudaMemcpyHostToDevice, pre));
    ISL_CUDA(e, cudaMemsetAsync(e->d_free_acc, 0, (size_t)n_batches * free_stride, pre));
    uint32_t epoch;
    if (int rc = next_epoch(e, &epoch)) return rc;
    // pre-pass of the tiles [t0, t1): defaults + free masks + histograms, then the stable partition into per-profile queues
    auto prepass = [&](uint32_t t0, uint32_t t1) -> int {
        k_prepare<<<t1 - t0, kTileThreads, 0, pre>>>(0, d_in, d_out, reinterpret_cast<uint32_t*>(e->d_occ.get()), e->G, e->lo, e->hi, e->prof,
                                                     e->d_tile_counts, e->d_ctrl, e->d_tiles, e->d_free_acc, free_stride / 4, t0);
        if (int rc = check_launch(e, "k_prepare")) return rc;
        if (timing) cudaEventRecord(e->ev[1], e->stream);
        k_partition<<<t1 - t0, kTileThreads, 0, pre>>>(0, d_in, e->prof.n, e->d_tile_counts, 0, e->cand_profiles, e->d_qall, e->d_cctl,
                                                       e->d_tiles, q_stride, t0);
        return check_launch(e, "k_partition");
    };
    // batch b of a fed stream: H2D of its requests, its pre-pass, its ready flag — all on the feed stream
    std::vector<uint32_t> batch_tile0(n_batches + 1, n_tiles_total);
    for (uint32_t t = n_tiles_total; t-- > 0;) batch_tile0[e->h_tiles[t].batch] = t;
    for (uint32_t b = n_batches; b-- > 0;) if (batch_tile0[b] == n_tiles_total) batch_tile0[b] = batch_tile0[b + 1];   // empty batch: no tiles
    uint64_t fed_off = 0;
    auto feed_batch = [&](uint32_t b) -> int {
        if (sizes[b]) {
            ISL_CUDA(e, cudaMemcpyAsync(const_cast<uint2*>(d_in) + fed_off, h_in + fed_off, (size_t)sizes[b] * sizeof(uint2), cudaMemcpyHostToDevice, pre));
            if (int rc = prepass(batch_tile0[b], batch_tile0[b + 1])) return rc;
        }
        k_set_flag<<<1, 1, 0, pre>>>(e->d_ready + b, epoch);
        fed_off += sizes[b];
        return check_launch(e, "k_set_flag");
    };
    if (timing) cudaEventRecord(e->ev[0], e->stream);
    if (feed) {
        if (int rc = feed_batch(0)) return rc;
        ISL_CUDA(e, cudaEventRecord(e->ev_feed, pre));                  // tables + first batch are on their way: the pipeline may start
        ISL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_feed, 0));
    } else if (int rc = prepass(0, n_tiles_total)) return rc;
    if (timing) cudaEventRecord(e->ev[2], e->stream);
    uint32_t* ring_done = nullptr;
    if (ring && window) {       // the owner's counters sit behind its result array; the other ranks reach them through the same peer mapping
        uint2* base = e->has_prev ? e->d_owner_out.get() : e->d_res.get();
        if (!base) return ISL_ESTATE;
        ring_done = reinterpret_cast<uint32_t*>(base + e->cfg.max_batch);
        if (!e->has_prev) ISL_CUDA(e, cudaMemsetAsync(ring_done, 0, (size_t)n_chunks * sizeof(uint32_t), e->stream));
    }
    const bool trace = e->cfg.flags & ISL_FLAG_TRACE;
    if (trace) {
        ISL_CUDA(e, e->d_trace.reserve((size_t)n_chunks * plan.n_seg, Growth::headroom));
        ISL_CUDA(e, cudaMemsetAsync(e->d_trace, 0, (size_t)n_chunks * plan.n_seg * kTraceWords * sizeof(unsigned long long), e->stream));
        e->trace_chunks = n_chunks; e->trace_seg = plan.n_seg;
    }
    if (plan.spec) if (int rc = prepare_spec(e, n_chunks, epoch, e->stream)) return rc;
    PipeArgs args = pipe_args(e, plan, n_chunks, epoch, q_stride, d_out);
    args.ready = feed ? e->d_ready.get() : nullptr; args.done_cnt = (h_out_dev || window) ? e->d_done_cnt.get() : nullptr; args.host_out = h_out_dev;
    args.copier = h_out_dev ? 1u : 0u; args.window = window; args.owner_out = ring ? e->d_owner_out.get() : nullptr;
    if (ring_done) { args.ring_done = ring_done; args.world = e->ring_world; }
    args.trace = trace ? e->d_trace.get() : nullptr;
    args.inbox = ring && e->has_prev ? e->d_inbox.get() : nullptr; args.outbox = ring ? e->d_outbox.get() : nullptr; args.xepoch = xepoch;
    if (plan.spec) {
        if (ring) {         // no token ring: the records themselves cross the ranks
            args.inbox = nullptr; args.outbox = nullptr;
            args.spec_world = e->spec_world; args.spec_rank = e->spec_rank; args.spec_base = e->lo / plan.seg; args.spec_total = ceil_div(e->G, plan.seg);
            for (uint32_t k = 0; k < e->spec_world; ++k) args.spec_peer[k] = e->spec_peer[k];
        }
        if (const char* v = getenv("ISL_SPEC_DBG")) {       // per-round stamps of one (chunk, stage) cell: tools/spec_trace.py
            unsigned cchunk = 0, cstage = 0;
            if (sscanf(v, "%u,%u", &cchunk, &cstage) == 2) {
                ISL_CUDA(e, e->d_specdbg.reserve(kSpecRounds));
                ISL_CUDA(e, cudaMemsetAsync(e->d_specdbg, 0, e->d_specdbg.bytes(), e->stream));
                args.spec_dbg = e->d_specdbg; args.spec_dbg_cell = (cchunk << 16) | cstage;
            }
        }
    }
    const int rc = start_pipeline(e, args);
    if (rc == ISL_ESTATE && ring) return ISL_ERANGE;    // a partitioned run cannot leave the pipeline: the token ring lives inside it
    if (rc == ISL_ESTATE) {         // the pre-pass above did not touch the occupancy (frees went to the free masks): redo batch by batch
        e->max_coresident = -1;     // and do not try the pipeline again on this engine
        if (feed) {                 // only batch 0 was fed: bring the whole stream in behind it
            ISL_CUDA(e, cudaEventRecord(e->ev_feed_done, pre));
            ISL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_feed_done, 0));
            ISL_CUDA(e, cudaMemcpyAsync(const_cast<uint2*>(d_in), h_in, (size_t)total * sizeof(uint2), cudaMemcpyHostToDevice, e->stream));
        }
        return run_batches(e, c, d_in, d_out, Path::chunks);
    }
    if (rc) return rc;
    if (feed) {     // the remaining batches, while the pipeline works on the first ones
        for (uint32_t b = 1; b < n_batches; ++b)
            if (int rc2 = feed_batch(b)) {
                // the resident pipeline would spin on ready[b] until its trap: publish 'closed' for every batch not fed so that it drains
                std::vector<uint32_t> closed(n_batches - b, ~epoch);
                cudaMemcpy(e->d_ready + b, closed.data(), closed.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
                cudaStreamSynchronize(e->stream);
                return rc2;
            }
        ISL_CUDA(e, cudaEventRecord(e->ev_feed_done, pre));
        ISL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_feed_done, 0));
        *delivered = h_out_dev != nullptr;
    }
    if (timing) {
        cudaEventRecord(e->ev[3], e->stream);
        cudaEventSynchronize(e->ev[3]);
        float t;
        cudaEventElapsedTime(&t, e->ev[0], e->ev[1]); e->st.ms_free += t;
        cudaEventElapsedTime(&t, e->ev[1], e->ev[2]); e->st.ms_partition += t;
        cudaEventElapsedTime(&t, e->ev[2], e->ev[3]); e->st.ms_commit += t;
        cudaEventElapsedTime(&t, e->ev[0], e->ev[3]); e->st.ms_total += t;
    }
    e->st.batches += n_batches;
    e->st.requests += total;
    return ISL_OK;
}

// One placement call: route(), then the executor of its path.  A device call only enqueues; a host call ends with its results delivered.
int run_stream(isl_engine* e, const Call& c) {
    uint64_t total = 0;
    uint32_t n_chunks = 0;
    for (uint32_t b = 0; b < c.n_batches; ++b) { total += c.sizes[b]; n_chunks += ceil_div(c.sizes[b], e->pipe_chunk); }
    if (total == 0) return ISL_OK;      // (every caller's Entry has checked total <= max_batch)
    Route r;
    if (int rc = route(e, c, total, n_chunks, &r)) return rc;
    const uint32_t n = c.sizes[0];
    if (c.src == Src::inline_host && (r.path == Path::few || r.path == Path::small)) {
        SmallReqs inl{};        // requests as kernel parameters, results into mapped pinned memory: 1 launch + 1 sync
        memcpy(inl.r, c.in, (size_t)n * sizeof(isl_request));
        if (int rc = r.path == Path::few ? run_few(e, n, inl, e->h_small_out.dev()) : run_small(e, n, nullptr, &inl, e->h_small_out.dev())) return rc;
        ISL_CUDA(e, cudaStreamSynchronize(e->stream));
        memcpy(c.out, e->h_small_out, (size_t)n * sizeof(isl_result));
        return ISL_OK;
    }
    const bool host = c.src != Src::device;
    const uint2* d_in = host ? e->d_req.get() : static_cast<const uint2*>(c.in);
    uint2* d_out = host ? e->d_res.get() : static_cast<uint2*>(c.out);
    if (host && !r.feed)        // one H2D copy up front; a fed stream copies batch by batch
        ISL_CUDA(e, cudaMemcpyAsync(e->d_req, c.in, (size_t)total * sizeof(isl_request), cudaMemcpyHostToDevice, e->stream));
    bool delivered = false;
    const int rc = r.path == Path::pipeline ? run_pipeline(e, c, r, d_in, d_out, total, n_chunks, &delivered)
                   : r.path == Path::small  ? run_small(e, n, d_in, nullptr, d_out)
                                            : run_batches(e, c, d_in, d_out, r.path);
    if (rc || !host) return rc;
    if (!delivered) ISL_CUDA(e, cudaMemcpyAsync(c.out, d_out, (size_t)total * sizeof(isl_result), cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

int place_batch_plain(isl_engine* e, uint32_t n, const isl_request* in, isl_result* out) {
    // One large batch that mixes profiles: the segment pipeline's decision loop (one launch for the chain of all segments, a shorter
    // loop per decision) beats the chunk path although nothing overlaps inside one chunk; a single placeable profile stays on the
    // chunk path, whose scan mode commits it without any chain.  A look at the profile bytes in host memory costs microseconds.
    bool mixed = false;
    if (n >= 4096) {
        uint32_t seen = 0;
        for (uint32_t i = 0; i < n && !mixed; ++i)
            if (in[i].op == ISL_OP_ALLOC && in[i].profile < ISL_MAX_PROFILES) { seen |= (1u << in[i].profile) & e->cand_profiles; mixed = (seen & (seen - 1)) != 0; }
    }
    return run_stream(e, Call{1, &n, n <= kSmallInline ? Src::inline_host : Src::host, in, out, 0, mixed});
}

// ISL_FLAG_ALL_NODES — the reference's literal multi-node behaviour (SURVEY Q5): Reconcile's node loop (:190-227) has no `break` after a
// successful node, so a pod is allocated on EVERY node that has capacity.  Nodes do not interact (an allocation on one node never
// changes what another node can take), so "every pod over all nodes" equals "every node over all pods": one restricted pass per node,
// each consuming capacity on its node; the record reported for a pod is the first node's (what the oracle's all_nodes switch reports).
// A compatibility mode for parity studies, one engine call per node — not a fast path.
int place_batch_locked(isl_engine* e, uint32_t n, const isl_request* in, isl_result* out) {
    if (!(e->cfg.flags & ISL_FLAG_ALL_NODES)) return place_batch_plain(e, n, in, out);
    const uint32_t n_nodes = (uint32_t)e->node_off.size() - 1;
    const auto [clo, chi] = storage_range(e, e->lo, e->hi);         // the caller's range, canonical
    RangeRestriction range{e, e->lo, e->hi};
    std::vector<isl_result> tmp(n);
    bool first = true;
    for (uint32_t k = 0; k < n_nodes; ++k) {
        const uint32_t node = e->prof.flip ? n_nodes - 1 - k : k;                  // nodes in policy order
        const uint32_t a = std::max(clo, e->node_off[node]), b = std::min(chi, e->node_off[node + 1]);
        if (a >= b) continue;
        range.set(a, b);
        if (int rc = place_batch_plain(e, n, in, first ? out : tmp.data())) return rc;
        if (!first)
            for (uint32_t i = 0; i < n; ++i)
                if (in[i].op == ISL_OP_ALLOC && out[i].status != ISL_ST_PLACED && tmp[i].status == ISL_ST_PLACED) out[i] = tmp[i];
        first = false;
    }
    return first ? place_batch_plain(e, n, in, out) : ISL_OK;      // empty range: defaults only
}

// Default row of every name (its size is what an unplaced ALLOC reports): the row of the first node, in canonical order, whose table has
// the name; without a node map (isl_set_node_tables) every node uses table 0.
void derive_default_rows(isl_engine* e) {
    for (uint32_t p = 0; p < e->prof.n; ++p) {
        e->prof.rows[p] = isl_profile{};
        if (e->node_table.empty()) {
            if (e->rows_all[0][p].n_starts) e->prof.rows[p] = e->rows_all[0][p];
            continue;
        }
        for (const uint8_t t : e->node_table)
            if (e->rows_all[t][p].n_starts) { e->prof.rows[p] = e->rows_all[t][p]; break; }
    }
}

// Every node back to table 0: no node map, the per-GPU table bytes zeroed, default rows from table 0 (isl_load_inventory, table reloads).
int reset_node_tables(isl_engine* e) {
    e->node_table.clear();
    ISL_CUDA(e, cudaMemsetAsync(e->d_gtab, 0, e->occ_bytes, e->stream));
    derive_default_rows(e);
    return ISL_OK;
}

constexpr uint32_t kSpecRingChunks = 64;         // chunks of one partitioned stream call that may speculate (17 MB of records per rank)

int spec_shared_alloc(isl_engine* e) {
    if (e->spec_shared) return ISL_OK;
    ISL_CUDA(e, e->d_spec.replace(kSpecRingChunks));
    ISL_CUDA(e, cudaMemset(e->d_spec, 0, e->d_spec.bytes()));
    e->spec_shared = true;
    return ISL_OK;
}

void spec_disconnect(isl_engine* e) {
    for (auto& peer : e->spec_peer) peer.reset();
    e->spec_world = 0;
}

// The argument checks of the stream entry points: 1..4096 batches that fit max_batch, buffers for a non-empty stream.  The engine's
// readiness is checked under the lock (Entry).
int stream_entry(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, bool have_buffers, uint64_t* total) {
    if (!e || !sizes || n_batches == 0 || n_batches > 4096) return ISL_EINVAL;
    *total = 0;
    for (uint32_t b = 0; b < n_batches; ++b) *total += sizes[b];
    if (*total && !have_buffers) return ISL_EINVAL;
    if (*total > e->cfg.max_batch) return ISL_ERANGE;
    return ISL_OK;
}

// device copy of the live occupancy (isl_snapshot_occupancy, isl_what_if)
int snapshot_occ(isl_engine* e) {
    ISL_CUDA(e, e->d_occ_snap.reserve(e->occ_bytes));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_occ_snap, e->d_occ, e->occ_bytes, cudaMemcpyDeviceToDevice, e->stream));
    return ISL_OK;
}

// CUDA IPC: the 64-byte handle of device memory p, and the mapping of a peer's handle into this process
int ipc_export(isl_engine* e, void* p, void* handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t h;
    ISL_CUDA(e, cudaIpcGetMemHandle(&h, p));
    memcpy(handle64, &h, sizeof h);
    return ISL_OK;
}

template <typename T>
int ipc_open(isl_engine* e, const void* handle64, T** out) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, sizeof h);
    void* p = nullptr;
    ISL_CUDA(e, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    *out = static_cast<T*>(p);
    return ISL_OK;
}

}  // namespace

extern "C" {

uint32_t isl_abi_version(void) { return ISL_ABI_VERSION; }

const char* isl_strerror(int code) {
    switch (code) {
        case ISL_OK: return "ok";
        case ISL_EINVAL: return "invalid argument or malformed table";
        case ISL_ENOMEM: return "out of memory";
        case ISL_ECUDA: return "CUDA error (see isl_last_cuda_error)";
        case ISL_ESTATE: return "profiles and inventory must be loaded first";
        case ISL_ERANGE: return "batch or inventory exceeds the engine's capacity";
        default: return "unknown error";
    }
}

const char* isl_last_cuda_error(const isl_engine* e) { return e ? e->cuda_err : "null engine"; }

int isl_create(const isl_config* cfg, isl_engine** out) {
    if (!cfg || !out) return ISL_EINVAL;
    *out = nullptr;
    if (cfg->abi_version != ISL_ABI_VERSION) return ISL_EINVAL;
    if (cfg->max_gpus == 0 || cfg->max_gpus > ISL_MAX_GPUS || cfg->max_batch == 0) return ISL_EINVAL;
    if (cfg->policy > ISL_POLICY_LEAST_ALLOCATED) return ISL_EINVAL;
    if (node_scoring(cfg->policy) && (cfg->flags & ISL_FLAG_ALL_NODES)) return ISL_EINVAL;     // a pod on every node: no node to choose
    if ((cfg->flags & ISL_FLAG_FIRST_AVAILABLE) && (cfg->flags & ISL_FLAG_ALL_NODES)) return ISL_EINVAL;     // A7: one pod, every node
    GangMode gang;
    if (int rc = gang_mode(cfg, &gang)) return rc;
    if (request_major(*cfg) && cfg->max_gpus > kBfMaxGpus) return ISL_ERANGE;
    if (cfg->quirks & ~ISL_QUIRKS_REF_EXACT) return ISL_EINVAL;
    isl_engine* e = new (std::nothrow) isl_engine;
    if (!e) return ISL_ENOMEM;
    e->cfg = *cfg;
    e->gang = gang;
    {   // pipeline chunk size: ISL_PIPE_CHUNK (requests, rounded to tiles) overrides the default
        uint32_t pc = kChunk;
        if (const char* v = getenv("ISL_PIPE_CHUNK")) pc = (uint32_t)strtoul(v, nullptr, 10);
        pc = std::max(kTile, std::min(kChunk, pc / kTile * kTile));
        e->pipe_chunk = pc;
    }
    if (const char* v = getenv("ISL_WAIT_SECONDS")) { const double sec = atof(v); if (sec > 0) e->wait_ns = (unsigned long long)(sec * 1e9); }
    int dev = cfg->device;
    if (dev < 0 && cudaGetDevice(&dev) != cudaSuccess) { delete e; return ISL_ECUDA; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || dev >= ndev) { delete e; return ISL_ECUDA; }
    e->device = dev;
    DeviceGuard guard(dev);
    // a half-built engine is deleted under the guard: its members free what was allocated so far on its device
#define ISL_TRY(call) do { if ((call) != cudaSuccess) { delete e; return ISL_ECUDA; } } while (0)
    ISL_TRY(cudaStreamCreateWithFlags(e->stream.out(), cudaStreamNonBlocking));
    {   // Load every kernel NOW.  With CUDA's lazy module loading the first launch of a kernel loads it, and that load can wait for the
        // device to drain — a fed host stream launches k_prepare / k_partition / k_set_flag for batch b WHILE the pipeline kernel is
        // spinning on ready[b]: a first-ever launch at that moment deadlocks (seen as the 20 s trap of a process whose first call was a
        // stream with an empty first batch).
        cudaFuncAttributes fa;
        const void* kernels[] = {(const void*)k_prepare, (const void*)k_partition, (const void*)k_set_flag, (const void*)k_few, (const void*)k_build_lut, (const void*)k_eval_starts,
                                 (const void*)k_free_spans, (const void*)k_capacity, (const void*)k_sweep_count, (const void*)k_sweep_scatter, (const void*)k_commit, (const void*)k_bestfit<false>, (const void*)k_bestfit<true>,
                                 (const void*)k_bestfit<false, true>, (const void*)k_bestfit<true, true>, (const void*)k_victim_map, (const void*)k_preempt, (const void*)k_nodefit<false>,
                                 (const void*)k_bestfit<false, false, true>, (const void*)k_bestfit<true, false, true>, (const void*)k_nodefit<true>,
                                 (const void*)k_chain<1>, (const void*)k_chain<2>, (const void*)k_chain<4>, (const void*)k_small<1>, (const void*)k_small<2>, (const void*)k_small<4>};
        const void* pipes[] = {(const void*)k_pipeline<1, false, false>, (const void*)k_pipeline<1, true, false>, (const void*)k_pipeline<2, false, false>, (const void*)k_pipeline<2, true, false>,
                               (const void*)k_pipeline<4, false, false>, (const void*)k_pipeline<4, true, false>,
                               (const void*)k_pipeline<1, false, true>, (const void*)k_pipeline<1, true, true>, (const void*)k_pipeline<2, false, true>, (const void*)k_pipeline<2, true, true>,
                               (const void*)k_pipeline<4, false, true>, (const void*)k_pipeline<4, true, true>};
        for (const void* k : kernels) ISL_TRY(cudaFuncGetAttributes(&fa, k));
        for (const void* k : pipes) ISL_TRY(cudaFuncGetAttributes(&fa, k));
        // dynamic shared memory opt-in, once per engine on its own device (a process-wide cache keyed by a truncated ordinal would
        // skip devices 8.. and race between threads)
        const void* chains[] = {(const void*)k_chain<1>, (const void*)k_chain<2>, (const void*)k_chain<4>};
        for (const void* k : chains) ISL_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kQCap * sizeof(uint16_t))));
        for (const void* k : {(const void*)k_bestfit<false>, (const void*)k_bestfit<false, true>, (const void*)k_bestfit<false, false, true>})
            ISL_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(256 * (kBfSmemGpus / 32 + kBfSmemGpus / 1024) * sizeof(uint32_t))));
        for (const void* k : pipes) ISL_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPipeSmem));
        for (const void* k : {(const void*)k_nodefit<false>, (const void*)k_nodefit<true>})
            ISL_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(ISL_MAX_PROFILES * (kNfSmemNodes + 64 + 32 + 32) * sizeof(uint32_t))));
        int optin = 0;          // k_preempt's share of the partition: up to what the device lets one CTA have
        ISL_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        ISL_TRY(cudaFuncGetAttributes(&fa, k_preempt));
        ISL_TRY(cudaFuncSetAttribute((const void*)k_preempt, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes));
        // each k_ganglocal instantiation (loaded here as well): its shares may have what the device lets one CTA have beside the
        // instantiation's own static words; the engine keeps the opt-in of the one it launches
        for (const GangKernel& k : kGangKernels) {
            ISL_TRY(cudaFuncGetAttributes(&fa, k.fn));
            ISL_TRY(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes));
            if (&k == e->gang.place) e->gn.optin = optin - (int)fa.sharedSizeBytes;
        }
        for (const GangKernel& k : kPreemptGangKernels) {     // and each k_preempt_gangs instantiation
            ISL_TRY(cudaFuncGetAttributes(&fa, k.fn));
            ISL_TRY(cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes));
            if (&k == e->gang.preempt) e->pre.optin = optin - (int)fa.sharedSizeBytes;
        }
    }
    e->occ_bytes = ((size_t)cfg->max_gpus + kSweepBlock - 1) / kSweepBlock * kSweepBlock;
    const uint32_t max_tiles = ceil_div(cfg->max_batch, kTile) + 4096;   // + one partial tile per batch of a stream
    ISL_TRY(e->d_occ.reserve(e->occ_bytes));
    ISL_TRY(e->d_lut.reserve(ISL_MAX_TABLES * ISL_MAX_PROFILES * 256));
    ISL_TRY(e->d_feas.reserve(ISL_MAX_TABLES * 256));
    ISL_TRY(cudaMemset(e->d_feas, 0, e->d_feas.bytes()));
    ISL_TRY(e->d_capn.reserve(ISL_MAX_TABLES * ISL_MAX_PROFILES * 256));
    ISL_TRY(e->d_seq.reserve(ISL_MAX_TABLES * ISL_MAX_PROFILES * 256));
    ISL_TRY(e->d_sizes.reserve(ISL_MAX_TABLES * ISL_MAX_PROFILES));
    ISL_TRY(e->d_score.reserve(ISL_MAX_TABLES * ISL_MAX_PROFILES * 256));
    ISL_TRY(e->d_cap.reserve(ISL_MAX_PROFILES));
    ISL_TRY(e->d_gtab.reserve(e->occ_bytes));
    ISL_TRY(cudaMemset(e->d_gtab, 0, e->occ_bytes));
    ISL_TRY(e->d_cand_o16.reserve(e->occ_bytes));
    ISL_TRY(e->d_req.reserve(cfg->max_batch));
    ISL_TRY(e->d_res.reserve((size_t)cfg->max_batch + kMaxStreamChunks * sizeof(uint32_t) / sizeof(uint2)));
    ISL_TRY(e->d_q.reserve(kQCap));
    ISL_TRY(e->d_tile_counts.reserve((size_t)max_tiles * ISL_MAX_PROFILES));
    ISL_TRY(e->d_cand.reserve(e->occ_bytes));
    ISL_TRY(e->d_log.reserve(kChunk));
    ISL_TRY(e->d_sweep_counts.reserve(e->occ_bytes / kSweepBlock));
    ISL_TRY(e->d_ctrl.reserve(1));
    ISL_TRY(cudaMemset(e->d_ctrl, 0, sizeof(Ctrl)));
    ISL_TRY(cudaMemset(e->d_occ, 0xFF, e->occ_bytes));
    for (auto& ev : e->ev) ISL_TRY(cudaEventCreate(ev.out()));
    ISL_TRY(e->h_small_out.reserve(kSmallInline));
#undef ISL_TRY
    *out = e;
    return ISL_OK;
}

int isl_destroy(isl_engine* e) {
    if (!e) return ISL_EINVAL;
    if (e->open.active) isl_stream_close(e);        // a persistent pipeline would never let the stream synchronise
    DeviceGuard guard(e->device);                   // the members release everything on the engine's device
    if (e->stream) cudaStreamSynchronize(e->stream);
    delete e;
    return ISL_OK;
}

int isl_set_stream(isl_engine* e, void* cuda_stream) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    if (e->stream) ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    if (cuda_stream) e->stream.borrow(static_cast<cudaStream_t>(cuda_stream));
    else ISL_CUDA(e, cudaStreamCreateWithFlags(e->stream.out(), cudaStreamNonBlocking));
    return ISL_OK;
}

int isl_synchronize(isl_engine* e) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

// The argument checks of isl_load_profiles (one table, every row must have placements) and isl_load_profile_tables, before the lock
static int check_tables(const isl_engine* e, uint32_t n_tables, uint32_t n, const isl_profile* rows, bool allow_absent) {
    if (!e || !rows || n == 0 || n > ISL_MAX_PROFILES || n_tables == 0 || n_tables > ISL_MAX_TABLES) return ISL_EINVAL;
    // Validate what would make the reference panic (SURVEY Q7): empty Placements (:334), start >= 8 (:345).
    uint32_t total_cand = 0;
    for (uint32_t r = 0; r < n_tables * n; ++r) {
        if (rows[r].n_starts == 0 && !allow_absent) return ISL_EINVAL;
        if (rows[r].n_starts > ISL_MAX_STARTS) return ISL_EINVAL;
        for (uint32_t k = 0; k < rows[r].n_starts; ++k) {
            if (rows[r].starts[k] >= ISL_SLOTS) return ISL_EINVAL;
            for (uint32_t j = 0; j < k; ++j) if (rows[r].starts[j] == rows[r].starts[k]) return ISL_EINVAL;   // shim de-duplicates
            total_cand += candidate_mask(rows[r].size, rows[r].starts[k], e->cfg.quirks) != 0;
        }
    }
    if (total_cand > kMaxCand) return ISL_EINVAL;          // more (table, profile, start) candidates than the chain's 4 x 32 lane slots
    return ISL_OK;
}

// The tables of both calls, under their Entry
static int load_tables(isl_engine* e, uint32_t n_tables, uint32_t n, const isl_profile* rows) {
    e->n_tables = n_tables;
    memset(e->rows_all, 0, sizeof(e->rows_all));
    for (uint32_t t = 0; t < n_tables; ++t) memcpy(e->rows_all[t], rows + (size_t)t * n, n * sizeof(isl_profile));
    e->prof.n = n; e->prof.quirks = e->cfg.quirks; e->prof.flip = reversed(e) ? e->G : 0u;
    memset(e->prof.rows, 0, sizeof(e->prof.rows));
    // new tables, new node map: every node uses table 0 until isl_set_node_tables names the tables again (a map kept from the old
    // tables could name a table that no longer exists, or one whose rows changed)
    if (int rc = reset_node_tables(e)) return rc;
    // chain candidates: every (table, profile, start) the search can ever return, in row order
    memset(&e->tab, 0, sizeof(e->tab));
    uint32_t c = 0; e->cand_profiles = 0;
    for (uint32_t t = 0; t < n_tables; ++t)
        for (uint32_t p = 0; p < n; ++p) {
            const isl_profile& row = e->rows_all[t][p];
            uint32_t ord = 0;
            for (uint32_t k = 0; k < row.n_starts; ++k) {
                const uint32_t m = candidate_mask(row.size, row.starts[k], e->cfg.quirks);
                if (!m) continue;
                e->tab.desc[c / 32][c % 32] = p | (ord << 4) | ((uint32_t)row.starts[k] << 7) | ((uint32_t)row.size << 11) | (m << 16) | (t << 24) | (1u << 31);
                ++c; ++ord;
                e->cand_profiles |= 1u << p;
            }
        }
    e->n_cand_slots = c <= 32 ? 1 : (c <= 64 ? 2 : 4);
    for (uint32_t t = 0; t < kMaxTables; ++t) {      // node scoring: a table's width in memory slices, the largest start + size of its rows
        e->nf.width[t] = 0;
        for (uint32_t p = 0; t < n_tables && p < n; ++p)
            for (uint32_t k = 0; k < e->rows_all[t][p].n_starts; ++k)
                e->nf.width[t] = std::max<uint8_t>(e->nf.width[t], e->rows_all[t][p].starts[k] + e->rows_all[t][p].size);
    }
    ISL_CUDA(e, cudaMemsetAsync(e->d_feas, 0, ISL_MAX_TABLES * 256 * sizeof(uint16_t), e->stream));
    for (uint32_t t = 0; t < n_tables; ++t) {
        DevProfiles dp{};
        dp.n = n; dp.quirks = e->cfg.quirks;
        memcpy(dp.rows, e->rows_all[t], sizeof(dp.rows));
        k_build_lut<<<1, 256, 0, e->stream>>>(dp, t, e->d_lut, e->d_feas, e->d_capn, e->d_seq);
        if (int rc = check_launch(e, "k_build_lut")) return rc;
    }
    {
        uint8_t sizes[ISL_MAX_TABLES * ISL_MAX_PROFILES] = {0};
        for (uint32_t t = 0; t < n_tables; ++t) for (uint32_t p = 0; p < n; ++p) sizes[t * ISL_MAX_PROFILES + p] = e->rows_all[t][p].size;
        ISL_CUDA(e, cudaMemcpyAsync(e->d_sizes, sizes, sizeof(sizes), cudaMemcpyHostToDevice, e->stream));
    }
    {   // what a best-fit family policy minimises, per table; zero for first-fit and right-to-left, whose gangs (isl_place_gangs) run
        // through the same kernel: its key is then the class minimum alone
        std::vector<uint8_t> score((size_t)ISL_MAX_TABLES * ISL_MAX_PROFILES * 256);      // the copy below completes before this function returns (stream sync)
        for (uint32_t t = 0; t < n_tables && bestfit_family(e->cfg.policy); ++t) {
            std::vector<uint32_t> cand;                              // every (profile, start) mask of the table the search can return
            for (uint32_t p = 0; p < n; ++p)
                for (uint32_t k = 0; k < e->rows_all[t][p].n_starts; ++k)
                    if (const uint32_t m = candidate_mask(e->rows_all[t][p].size, e->rows_all[t][p].starts[k], e->cfg.quirks)) cand.push_back(m);
            for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p)
                for (uint32_t o = 0; o < 256; ++o) {
                    uint32_t mine = 0;                                   // the mask the profile would take there: first legal start in row order
                    if (p < n)
                        for (uint32_t k = 0; k < e->rows_all[t][p].n_starts && !mine; ++k) {
                            const uint32_t m = candidate_mask(e->rows_all[t][p].size, e->rows_all[t][p].starts[k], e->cfg.quirks);
                            if (m && (o & m) == 0) mine = m;
                        }
                    // ISL_POLICY_BEST_FIT: free slices of the GPU AFTER the placement, fewest first (with several tables one name may
                    // span different sizes, so "after" is not "before minus a constant")
                    uint32_t v = 8u - (uint32_t)__builtin_popcount(o | mine);
                    if (e->cfg.policy == ISL_POLICY_MIN_FRAG) {
                        v = 0;
                        if (mine) for (uint32_t m : cand) v += ((o & m) == 0) && (((o | mine) & m) != 0);      // pairs that stop being feasible
                    }
                    score[((size_t)t * ISL_MAX_PROFILES + p) * 256 + o] = (uint8_t)v;
                }
        }
        ISL_CUDA(e, cudaMemcpyAsync(e->d_score, score.data(), score.size(), cudaMemcpyHostToDevice, e->stream));
    }
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->have_profiles = true;
    return ISL_OK;
}

int isl_load_profiles(isl_engine* e, uint32_t n, const isl_profile* rows) {
    if (int rc = check_tables(e, 1, n, rows, false)) return rc;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    return load_tables(e, 1, n, rows);
}

int isl_load_profile_tables(isl_engine* e, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows) {
    if (int rc = check_tables(e, n_tables, n_profiles, rows, true)) return rc;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    return load_tables(e, n_tables, n_profiles, rows);
}

int isl_set_node_tables(isl_engine* e, uint32_t n_nodes, const uint8_t* table_of_node) {
    if (!e || !table_of_node) return ISL_EINVAL;
    Entry guard(e, Needs::ready);
    if (guard.rc) return guard.rc;
    if (n_nodes + 1 != e->node_off.size()) return ISL_EINVAL;
    for (uint32_t n = 0; n < n_nodes; ++n) if (table_of_node[n] >= e->n_tables) return ISL_EINVAL;
    e->node_table.assign(table_of_node, table_of_node + n_nodes);
    std::vector<uint8_t> gtab(e->G);
    for (uint32_t n = 0; n < n_nodes; ++n)
        for (uint32_t g = e->node_off[n]; g < e->node_off[n + 1]; ++g) gtab[flip_gpu(g, e->prof.flip)] = table_of_node[n];
    ISL_CUDA(e, cudaMemcpyAsync(e->d_gtab, gtab.data(), e->G, cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    derive_default_rows(e);
    return ISL_OK;
}

int isl_load_inventory(isl_engine* e, uint32_t n_nodes, const uint32_t* node_off, const uint8_t* occ) {
    if (!e || !node_off || n_nodes == 0) return ISL_EINVAL;
    if (node_off[0] != 0) return ISL_EINVAL;
    for (uint32_t i = 0; i < n_nodes; ++i) if (node_off[i + 1] < node_off[i]) return ISL_EINVAL;
    const uint32_t G = node_off[n_nodes];
    if (G == 0 || !occ) return ISL_EINVAL;
    if (G > e->cfg.max_gpus) return ISL_ERANGE;
    // k_nodefit's min-trees have kNfMaxLevels levels over the nodes of a range, empty nodes included: refused here, before the guard,
    // so that the previous inventory stays in place and an accepted inventory can always be placed on
    if (node_scoring(e->cfg.policy) && n_nodes > kNfMaxNodes) return ISL_ERANGE;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->node_off.assign(node_off, node_off + n_nodes + 1);
    e->G = G; e->lo = 0; e->hi = G;
    e->prof.flip = reversed(e) ? G : 0u;      // ISL_POLICY_RIGHT_TO_LEFT: the inventory is stored in reverse canonical order
    e->snap_G = 0;                  // a snapshot belongs to the inventory it was taken from
    ISL_CUDA(e, cudaMemsetAsync(e->d_occ, 0xFF, e->occ_bytes, e->stream));
    if (int rc = reset_node_tables(e)) return rc;      // every node uses table 0 until isl_set_node_tables
    std::vector<uint8_t> rev;
    if (e->prof.flip) { rev.assign(occ, occ + G); std::reverse(rev.begin(), rev.end()); occ = rev.data(); }
    ISL_CUDA(e, cudaMemcpyAsync(e->d_occ, occ, G, cudaMemcpyHostToDevice, e->stream));
    if (node_scoring(e->cfg.policy)) {      // k_nodefit finds the nodes of a range through them
        ISL_CUDA(e, e->nf.node_off.replace((size_t)n_nodes + 1));
        ISL_CUDA(e, cudaMemcpyAsync(e->nf.node_off, node_off, ((size_t)n_nodes + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    }
    if (e->gang.place || e->gang.preempt) {
        // k_ganglocal and k_preempt_gangs walk the nodes in storage order (reversed under right-to-left)
        auto& off = e->gn.off;
        off.assign(node_off, node_off + n_nodes + 1);
        if (e->prof.flip) { std::reverse(off.begin(), off.end()); for (auto& x : off) x = G - x; }
        ISL_CUDA(e, e->gn.node_off.replace((size_t)n_nodes + 1));
        ISL_CUDA(e, cudaMemcpyAsync(e->gn.node_off, off.data(), ((size_t)n_nodes + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    }
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->have_inventory = true;
    return ISL_OK;
}

int isl_read_occupancy(isl_engine* e, uint8_t* out) {
    if (!e || !out) return ISL_EINVAL;
    Entry guard(e, Needs::inventory);
    if (guard.rc) return guard.rc;
    ISL_CUDA(e, cudaMemcpyAsync(out, e->d_occ, e->G, cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    if (e->prof.flip) std::reverse(out, out + e->G);       // canonical order at the boundary
    return ISL_OK;
}

int isl_write_occupancy(isl_engine* e, uint32_t first_gpu, uint32_t n, const uint8_t* occ) {
    if (!e || (n && !occ)) return ISL_EINVAL;
    Entry guard(e, Needs::inventory);
    if (guard.rc) return guard.rc;
    if ((uint64_t)first_gpu + n > e->G) return ISL_ERANGE;
    if (n == 0) return ISL_OK;
    std::vector<uint8_t> rev;
    if (e->prof.flip) { rev.assign(occ, occ + n); std::reverse(rev.begin(), rev.end()); occ = rev.data(); first_gpu = e->G - first_gpu - n; }
    ISL_CUDA(e, cudaMemcpyAsync(e->d_occ + first_gpu, occ, n, cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

int isl_snapshot_occupancy(isl_engine* e) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::inventory);
    if (guard.rc) return guard.rc;
    if (int rc = snapshot_occ(e)) return rc;
    e->snap_G = e->G;
    return ISL_OK;
}

int isl_restore_occupancy(isl_engine* e) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::inventory);
    if (guard.rc) return guard.rc;
    if (!e->d_occ_snap || e->snap_G != e->G) return ISL_ESTATE;     // a snapshot belongs to the inventory it was taken from
    ISL_CUDA(e, cudaMemcpyAsync(e->d_occ, e->d_occ_snap, e->occ_bytes, cudaMemcpyDeviceToDevice, e->stream));
    return ISL_OK;
}

uint32_t isl_num_gpus(const isl_engine* e) { return e ? e->G : 0; }

uint32_t isl_gpu_to_node(const isl_engine* e, uint32_t gpu) {
    if (!e || gpu >= e->G) return ISL_GPU_NONE;
    auto it = std::upper_bound(e->node_off.begin(), e->node_off.end(), gpu);
    return (uint32_t)(it - e->node_off.begin()) - 1;
}

int isl_place_batch(isl_engine* e, uint32_t n, const isl_request* in, isl_result* out) {
    if (!e || (n && (!in || !out))) return ISL_EINVAL;
    Entry guard(e, Needs::ready, n);
    if (guard.rc) return guard.rc;
    if (n == 0) return ISL_OK;
    return place_batch_locked(e, n, in, out);
}

int isl_place_batch_range(isl_engine* e, uint32_t lo, uint32_t hi, uint32_t n, const isl_request* in, isl_result* out) {
    if (!e || (n && (!in || !out))) return ISL_EINVAL;
    Entry guard(e, Needs::ready, n);                // restriction, placement and restore under ONE lock: two callers cannot interleave
    if (guard.rc) return guard.rc;
    if (lo > hi || hi > e->G) return ISL_EINVAL;
    if (n == 0) return ISL_OK;
    RangeRestriction range{e, e->lo, e->hi};
    range.set(lo, hi);
    return place_batch_locked(e, n, in, out);
}

int isl_place_gangs(isl_engine* e, uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out) {
    if (!e || (n_gangs && !gang_off)) return ISL_EINVAL;
    if (gang_off && gang_off[0] != 0) return ISL_EINVAL;
    for (uint32_t i = 0; i < n_gangs; ++i) if (gang_off[i + 1] <= gang_off[i]) return ISL_EINVAL;      // no empty gang
    const uint32_t n = n_gangs ? gang_off[n_gangs] : 0;
    if (n && (!in || !out)) return ISL_EINVAL;
    // one pod on every node with capacity has no all-or-nothing meaning; gangs under node scoring only on an ISL_FLAG_GANG_NODE_SCORE engine
    const GangMode& m = e->gang;
    if (m.gangs_refused) return ISL_EINVAL;
    // per-gang bytes: each gang's locality (L1, L4), the engine's under ISL_FLAG_GANG_MIN_MEMBERS without ISL_FLAG_GANG_LOCALITY, and its
    // m' (M1, M6); 0 for a gang without ALLOCs
    const bool per_gang = m.locality == kLocPerGang;
    std::vector<uint8_t> locality;
    std::vector<uint32_t> min_members;
    if (per_gang || m.min_members) {
        locality.assign(n_gangs, (uint8_t)(per_gang ? ISL_GANG_ANY_NODES : m.locality));
        min_members.assign(m.min_members ? n_gangs : 0, 0);
        for (uint32_t i = 0; i < n_gangs; ++i) {
            const uint32_t r0 = gang_off[i], r1 = gang_off[i + 1];
            // B1: bytes 4..255 are balanced gangs on an ISL_FLAG_GANG_BALANCED engine.  N6: few-node gangs are not node-scored, unless
            // the engine scores every gang kind (C2)
            if (per_gang && (alloc_shared(in, r0, r1, [&](uint32_t r) { return in[r].start; }, &locality[i]) < 0 ||
                             (locality[i] > ISL_GANG_DISTINCT_NODES && !m.balanced) ||
                             (locality[i] == ISL_GANG_FEW_NODES && m.node_score && !m.score_all))) return ISL_EINVAL;
            if (m.min_members) {
                uint8_t size = 0;
                const int64_t k = alloc_shared(in, r0, r1, [&](uint32_t r) { return in[r].size; }, &size);
                if (k < 0) return ISL_EINVAL;
                min_members[i] = (size == 0 || size >= k) ? (uint32_t)k : size;
            }
        }
    }
    if (n > e->cfg.max_batch) return ISL_ERANGE;
    Entry guard(e, Needs::ready, n);
    if (guard.rc) return guard.rc;
    if (n == 0) return ISL_OK;
    if (e->hi == e->lo || e->hi - e->lo > kBfMaxGpus) return ISL_ERANGE;          // the class bitmaps of k_bestfit
    const size_t min_at = ((size_t)n_gangs + 1) * sizeof(uint32_t) + ((locality.size() + 3) & ~(size_t)3);     // m' after the bytes
    ISL_CUDA(e, e->d_scratch.reserve(min_at + min_members.size() * sizeof(uint32_t)));
    uint32_t* d_gang_off = reinterpret_cast<uint32_t*>(e->d_scratch.get());
    const uint8_t* d_locality = reinterpret_cast<const uint8_t*>(d_gang_off + n_gangs + 1);      // the bytes right after the offsets
    ISL_CUDA(e, cudaMemcpyAsync(d_gang_off, gang_off, ((size_t)n_gangs + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    if (!locality.empty())
        ISL_CUDA(e, cudaMemcpyAsync((void*)d_locality, locality.data(), locality.size(), cudaMemcpyHostToDevice, e->stream));
    if (!min_members.empty())
        ISL_CUDA(e, cudaMemcpyAsync((uint8_t*)e->d_scratch.get() + min_at, min_members.data(), min_members.size() * sizeof(uint32_t),
                                    cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_req, in, (size_t)n * sizeof(isl_request), cudaMemcpyHostToDevice, e->stream));
    if (int rc = m.place ? run_ganglocal(e, n_gangs, d_gang_off, d_locality, n, e->d_req, e->d_res)
                         : run_gangs(e, n_gangs, d_gang_off, n, e->d_req, e->d_res)) return rc;
    ISL_CUDA(e, cudaMemcpyAsync(out, e->d_res, (size_t)n * sizeof(isl_result), cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

// isl_preempt on an ISL_FLAG_GANG_PREEMPT engine, after k_victim_map: one cooperative launch of the engine's k_preempt_gangs
// instantiation on gang_layout's shares (kPgBytesPerGpu per GPU, in p.state when they do not fit in shared memory).  The gang offsets
// and the locality bytes go to p.gangs; every evict row starts as ISL_GPU_NONE.
int run_preempt_gangs(isl_engine* e, const std::vector<uint32_t>& gang_off, const std::vector<uint8_t>& locality, uint32_t n,
                      const uint8_t* d_prio, const uint8_t* d_masks) {
    auto& p = e->pre;
    const uint32_t n_gangs = (uint32_t)gang_off.size() - 1, Gr = e->hi - e->lo;
    const GangKernel& k = *e->gang.preempt;
    ISL_CUDA(e, p.gangs.reserve(gang_off.size() + (locality.size() + 3) / 4));
    uint32_t* d_gang_off = p.gangs;
    const uint8_t* d_locality = reinterpret_cast<const uint8_t*>(d_gang_off + gang_off.size());
    ISL_CUDA(e, cudaMemcpyAsync(d_gang_off, gang_off.data(), gang_off.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    if (!locality.empty())
        ISL_CUDA(e, cudaMemcpyAsync((void*)d_locality, locality.data(), locality.size(), cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, p.log.reserve(n));
    GangNodeArgs a;
    uint32_t grid, nodes;
    size_t smem;
    if (int rc = gang_layout(e, k.fn, p.optin, kPgBytesPerGpu, n_gangs, d_gang_off, e->d_req, e->d_res, a, &grid, &smem, &nodes)) return rc;
    if (!smem) ISL_CUDA(e, p.state.reserve((size_t)Gr * kPgBytesPerGpu));
    a.scratch = p.state;
    PreemptArgs pa{};
    pa.in = e->d_req; pa.prio = d_prio; pa.victims = p.victims; pa.vmap = p.vmap; pa.occ = e->d_occ; pa.gtab = e->d_gtab; pa.masks = d_masks;
    pa.out = e->d_res; pa.evict = p.evict;
    pa.n = n; pa.lo = e->lo; pa.Gr = Gr; pa.per_cta = a.share;      // GPUs per array of a share in shared memory, 0 = global memory
    a.share = 0;                                                    // NodeShare copies no occupancy byte: the kernel keeps its own state
    ISL_CUDA(e, p.keys.reserve((size_t)2 * grid));
    pa.keys = p.keys;
    ISL_CUDA(e, cudaMemsetAsync(p.evict, 0xFF, (size_t)n * ISL_SLOTS * sizeof(uint32_t), e->stream));
    PgLog* log = p.log;
    void* params[] = {&a, &pa, &e->prof, &log, &d_locality};
    return launch_cooperative(e, k.fn, k.name, grid, kGnThreads, smem, params);
}

int isl_preempt(isl_engine* e, uint32_t n, const isl_request* in, const uint8_t* priority,
                uint32_t n_victims, const isl_victim* victims, isl_result* out, uint32_t* evict) {
    if (!e || (n && (!in || !priority || !out || !evict)) || (n_victims && !victims)) return ISL_EINVAL;
    if (e->cfg.flags & ISL_FLAG_ALL_NODES) return ISL_EINVAL;      // one pod on every node with capacity: no single GPU to evict on
    for (uint32_t i = 0; i < n; ++i) if (in[i].op == ISL_OP_FREE) return ISL_EINVAL;      // releases are expressed by the victim list
    const bool gangs = e->gang.preempt;
    std::vector<uint32_t> gang_off;                                 // P1: maximal runs of equal handles
    std::vector<uint8_t> locality;                                  // under ISL_FLAG_GANG_LOCALITY: each gang's byte, 0 without ALLOCs
    if (gangs) {
        const bool per_gang = e->gang.locality == kLocPerGang;
        for (uint32_t i = 0; i < n; ++i)
            if (i == 0 || in[i].handle != in[i - 1].handle) gang_off.push_back(i);
        gang_off.push_back(n);
        if (per_gang) locality.assign(gang_off.size() - 1, (uint8_t)ISL_GANG_ANY_NODES);
        for (size_t g = 0; g + 1 < gang_off.size(); ++g) {
            const uint32_t r0 = gang_off[g], r1 = gang_off[g + 1];
            // P1: one priority byte per gang, and under ISL_FLAG_GANG_LOCALITY one locality byte, 0, 1 or 3
            uint8_t prio = 0;
            if (alloc_shared(in, r0, r1, [&](uint32_t r) { return priority[r]; }, &prio) < 0) return ISL_EINVAL;
            if (per_gang && (alloc_shared(in, r0, r1, [&](uint32_t r) { return in[r].start; }, &locality[g]) < 0 ||
                             (locality[g] != ISL_GANG_ANY_NODES && locality[g] != ISL_GANG_ONE_NODE &&
                              locality[g] != ISL_GANG_DISTINCT_NODES))) return ISL_EINVAL;
        }
    }
    if (n > e->cfg.max_batch || (uint64_t)n_victims > (uint64_t)ISL_SLOTS * e->cfg.max_gpus) return ISL_ERANGE;
    Entry guard(e, Needs::ready, n);
    if (guard.rc) return guard.rc;
    if (n == 0) return ISL_OK;
    const uint32_t Gr = e->hi - e->lo;
    if (Gr == 0 || Gr > kPreMaxGpus) return ISL_ERANGE;
    // one CTA per SM at most (the grid-wide exchange per preemptor is cheaper with fewer CTAs), at least one thread per GPU below that
    int sms = 0, per_sm = 0;
    ISL_CUDA(e, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, e->device));
    const uint32_t grid = std::max(1u, std::min((uint32_t)sms, ceil_div(Gr, kPreThreads))), per_cta = ceil_div(Gr, grid);
    const size_t smem = (size_t)per_cta * kPreBytesPerGpu;
    if (!gangs && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_preempt, kPreThreads, smem) != cudaSuccess || per_sm < 1)) {
        cudaGetLastError();
        return ISL_ERANGE;                                  // a share too large for one CTA's shared memory on this device
    }
    auto& p = e->pre;
    constexpr size_t kMaskBytes = kMaxTables * ISL_MAX_PROFILES * ISL_MAX_STARTS;
    ISL_CUDA(e, p.vmap.reserve((size_t)Gr * ISL_SLOTS));
    ISL_CUDA(e, p.evict.reserve((size_t)n * ISL_SLOTS));
    ISL_CUDA(e, p.err.reserve(1));
    ISL_CUDA(e, p.victims.reserve(std::max(n_victims, 1u)));
    ISL_CUDA(e, p.stage.reserve(kMaskBytes + n));
    ISL_CUDA(e, p.keys.reserve((size_t)2 * grid));
    uint8_t masks[kMaskBytes] = {0};                        // [table][profile][position in the row]: the start search's legal masks
    for (uint32_t t = 0; t < e->n_tables; ++t)
        for (uint32_t q = 0; q < e->prof.n; ++q)
            for (uint32_t k = 0; k < e->rows_all[t][q].n_starts; ++k)
                masks[(t * ISL_MAX_PROFILES + q) * ISL_MAX_STARTS + k] = (uint8_t)candidate_mask(e->rows_all[t][q].size, e->rows_all[t][q].starts[k], e->cfg.quirks);
    ISL_CUDA(e, cudaMemcpyAsync(e->d_req, in, (size_t)n * sizeof(isl_request), cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, cudaMemcpyAsync(p.stage, masks, kMaskBytes, cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, cudaMemcpyAsync(p.stage + kMaskBytes, priority, n, cudaMemcpyHostToDevice, e->stream));
    ISL_CUDA(e, cudaMemsetAsync(p.vmap, 0xFF, (size_t)Gr * ISL_SLOTS * sizeof(uint32_t), e->stream));
    ISL_CUDA(e, cudaMemsetAsync(p.err, 0, sizeof(uint32_t), e->stream));
    if (n_victims) {
        ISL_CUDA(e, cudaMemcpyAsync(p.victims, victims, (size_t)n_victims * sizeof(isl_victim), cudaMemcpyHostToDevice, e->stream));
        k_victim_map<<<ceil_div(n_victims, 256), 256, 0, e->stream>>>(n_victims, p.victims, e->d_occ, e->G, e->lo, e->hi, e->prof.flip, p.vmap, p.err);
        if (int rc = check_launch(e, "k_victim_map")) return rc;
        uint32_t err = 0;
        ISL_CUDA(e, cudaMemcpyAsync(&err, p.err, sizeof err, cudaMemcpyDeviceToHost, e->stream));
        ISL_CUDA(e, cudaStreamSynchronize(e->stream));
        if (err) return ISL_EINVAL;                         // a malformed, free or overlapping victim: nothing else runs
    }
    if (gangs) {
        if (int rc = run_preempt_gangs(e, gang_off, locality, n, p.stage + kMaskBytes, p.stage)) return rc;
    } else {
        PreemptArgs a{};
        a.in = e->d_req; a.prio = p.stage + kMaskBytes; a.victims = p.victims; a.vmap = p.vmap; a.occ = e->d_occ; a.gtab = e->d_gtab;
        a.masks = p.stage; a.out = e->d_res; a.evict = p.evict; a.keys = p.keys;
        a.n = n; a.lo = e->lo; a.Gr = Gr; a.per_cta = per_cta;
        void* params[] = {&a, &e->prof};
        if (int rc = launch_cooperative(e, (const void*)k_preempt, "k_preempt", grid, kPreThreads, smem, params)) return rc;
    }
    ISL_CUDA(e, cudaMemcpyAsync(out, e->d_res, (size_t)n * sizeof(isl_result), cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaMemcpyAsync(evict, p.evict, (size_t)n * ISL_SLOTS * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

int isl_place_stream(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, const isl_request* in, isl_result* out) {
    uint64_t total;
    if (int rc = stream_entry(e, n_batches, sizes, in && out, &total)) return rc;
    Entry guard(e, Needs::ready, total);
    if (guard.rc) return guard.rc;
    const int rc = run_stream(e, Call{n_batches, sizes, Src::host, in, out});
    if (rc && e->feed_stream) cudaStreamSynchronize(e->feed_stream);
    return rc;
}

int isl_place_stream_device(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, const void* d_in, void* d_out) {
    if (!d_in || !d_out) return ISL_EINVAL;
    uint64_t total;
    if (int rc = stream_entry(e, n_batches, sizes, true, &total)) return rc;
    Entry guard(e, Needs::ready, total);
    if (guard.rc) return guard.rc;
    return run_stream(e, Call{n_batches, sizes, Src::device, d_in, d_out});
}

int isl_ipc_inbox_handle(isl_engine* e, void* handle64) {
    if (!e || !handle64) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    bool fresh;
    ISL_CUDA(e, e->d_inbox.reserve(kMaxStreamChunks, Growth::exact, &fresh));
    if (fresh) ISL_CUDA(e, cudaMemset(e->d_inbox, 0, e->d_inbox.bytes()));
    return ipc_export(e, e->d_inbox, handle64);
}

int isl_ipc_connect(isl_engine* e, const void* next_handle64, int has_prev) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->d_outbox.reset();
    if (next_handle64) if (int rc = ipc_open(e, next_handle64, e->d_outbox.out())) return rc;
    e->has_prev = has_prev != 0;
    if (e->has_prev && !e->d_inbox) return ISL_ESTATE;
    return ISL_OK;
}

int isl_connect_local(isl_engine* e, isl_engine* next, int has_prev) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->d_outbox.reset();
    if (next) {
        if (!next->d_inbox) return ISL_ESTATE;
        e->d_outbox.borrow(next->d_inbox);
    }
    e->has_prev = has_prev != 0;
    if (e->has_prev && !e->d_inbox) return ISL_ESTATE;
    return ISL_OK;
}

// ---- speculative rounds over a partitioned inventory: every rank's record memory mapped into every other rank ------------------------
int isl_ipc_spec_handle(isl_engine* e, void* handle64) {
    if (!e || !handle64) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    if (int rc = spec_shared_alloc(e)) return rc;
    return ipc_export(e, e->d_spec, handle64);
}

// handles: world x 64 bytes (isl_ipc_spec_handle of every rank, own entry ignored); bounds: world + 1 canonical GPU indices, rank r owns
// [bounds[r], bounds[r + 1]).  world = 0 disconnects.
int isl_ipc_connect_spec(isl_engine* e, uint32_t world, uint32_t rank, const void* handles, const uint32_t* bounds) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    spec_disconnect(e);
    if (world == 0) return ISL_OK;
    if (world < 2 || world > 8 || rank >= world || !handles || !bounds) return ISL_EINVAL;
    if (int rc = spec_shared_alloc(e)) return rc;
    for (uint32_t r = 0; r < world; ++r) {
        if (r == rank) e->spec_peer[r].borrow(e->d_spec);
        else if (int rc = ipc_open(e, static_cast<const char*>(handles) + 64 * r, e->spec_peer[r].out())) return rc;
    }
    for (uint32_t r = 0; r <= world; ++r) e->spec_bounds[r] = bounds[r];
    e->spec_world = world; e->spec_rank = rank;
    return ISL_OK;
}

// same-process engines (tests: several ranks on one GPU)
int isl_connect_spec_local(isl_engine* e, uint32_t world, uint32_t rank, isl_engine* const* engines, const uint32_t* bounds) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    spec_disconnect(e);
    if (world == 0) return ISL_OK;
    if (world < 2 || world > 8 || rank >= world || !engines || !bounds) return ISL_EINVAL;
    if (int rc = spec_shared_alloc(e)) return rc;
    for (uint32_t r = 0; r < world; ++r) {
        if (r != rank && (!engines[r] || !engines[r]->spec_shared)) return ISL_ESTATE;     // every engine allocates first (isl_ipc_spec_handle)
        e->spec_peer[r].borrow(r == rank ? e->d_spec.get() : engines[r]->d_spec.get());
    }
    for (uint32_t r = 0; r <= world; ++r) e->spec_bounds[r] = bounds[r];
    e->spec_world = world; e->spec_rank = rank;
    return ISL_OK;
}

int isl_place_stream_partitioned(isl_engine* e, uint32_t n_batches, const uint32_t* sizes, const void* d_in, void* d_out, uint32_t stream_id) {
    if (!d_in || !d_out || stream_id == 0) return ISL_EINVAL;
    uint64_t total;
    if (int rc = stream_entry(e, n_batches, sizes, true, &total)) return rc;
    Entry guard(e, Needs::ready, total);
    if (guard.rc) return guard.rc;
    if (total == 0) return ISL_OK;
    if (request_major(e->cfg) || reversed(e)) return ISL_EINVAL;         // request-major / right-to-left policies do not partition
    return run_stream(e, Call{n_batches, sizes, Src::device, d_in, d_out, stream_id});
}

int isl_place_batch_device(isl_engine* e, uint32_t n, const void* d_in, void* d_out) {
    if (!e || (n && (!d_in || !d_out))) return ISL_EINVAL;
    Entry guard(e, Needs::ready, n);
    if (guard.rc) return guard.rc;
    return run_stream(e, Call{1, &n, Src::device, d_in, d_out});
}

int isl_place_batch_partitioned(isl_engine* e, uint32_t n, const void* d_in, void* d_out, const void* d_heads_in, void* d_heads_out) {
    if (!e || (n && (!d_in || !d_out)) || !d_heads_out) return ISL_EINVAL;
    Entry guard(e, Needs::ready, n);
    if (guard.rc) return guard.rc;
    if (n == 0) return ISL_OK;
    if (request_major(e->cfg) || reversed(e)) return ISL_EINVAL;         // request-major / right-to-left policies do not partition
    return run_chunks(e, n, static_cast<const uint2*>(d_in), static_cast<uint2*>(d_out), static_cast<const uint32_t*>(d_heads_in),
                      static_cast<uint32_t*>(d_heads_out));
}

int isl_set_partition(isl_engine* e, uint32_t lo, uint32_t hi) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::inventory);
    if (guard.rc) return guard.rc;
    if (lo > hi || hi > e->G) return ISL_EINVAL;
    std::tie(e->lo, e->hi) = storage_range(e, lo, hi);
    return ISL_OK;
}

void* isl_device_occupancy(isl_engine* e) { return e ? e->d_occ.get() : nullptr; }

int isl_free_batch(isl_engine* e, uint32_t n, const isl_span* spans) {
    if (!e || (n && !spans)) return ISL_EINVAL;
    Entry guard(e, Needs::inventory);
    if (guard.rc) return guard.rc;
    if (n == 0) return ISL_OK;
    ISL_CUDA(e, e->d_scratch.reserve((size_t)n * sizeof(isl_span)));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_scratch, spans, (size_t)n * sizeof(isl_span), cudaMemcpyHostToDevice, e->stream));
    k_free_spans<<<ceil_div(n, 256), 256, 0, e->stream>>>(n, reinterpret_cast<const isl_span*>(e->d_scratch.get()), reinterpret_cast<uint32_t*>(e->d_occ.get()),
                                                          e->G, e->lo, e->hi, e->d_ctrl, e->prof.flip);
    if (int rc = check_launch(e, "k_free_spans")) return rc;
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

int isl_eval_starts(isl_engine* e, uint32_t profile, uint32_t n, const uint8_t* occ, uint8_t* out) {
    if (!e || (n && (!occ || !out))) return ISL_EINVAL;
    Entry guard(e, Needs::profiles);
    if (guard.rc) return guard.rc;
    const uint32_t table = profile >> 8;
    profile &= 0xFFu;
    if (profile >= e->prof.n || table >= e->n_tables) return ISL_EINVAL;
    if (n == 0) return ISL_OK;
    ISL_CUDA(e, e->d_scratch.reserve((size_t)n * 2));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_scratch, occ, n, cudaMemcpyHostToDevice, e->stream));
    k_eval_starts<<<std::min(ceil_div(n, 256), 1184u), 256, 0, e->stream>>>(e->d_lut + (size_t)table * ISL_MAX_PROFILES * 256, profile, n, e->d_scratch, e->d_scratch + n);
    if (int rc = check_launch(e, "k_eval_starts")) return rc;
    ISL_CUDA(e, cudaMemcpyAsync(out, e->d_scratch + n, n, cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

int isl_read_trace(isl_engine* e, uint64_t* out, uint32_t max_words, uint32_t* n_chunks, uint32_t* n_seg) {
    if (!e || !n_chunks || !n_seg) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    *n_chunks = e->trace_chunks; *n_seg = e->trace_seg;
    const size_t words = (size_t)e->trace_chunks * e->trace_seg * kTraceWords;
    if (!out || words == 0) return ISL_OK;
    if (words > max_words) return ISL_ERANGE;
    ISL_CUDA(e, cudaMemcpyAsync(out, e->d_trace, words * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

int isl_get_stats(isl_engine* e, isl_stats* out) {
    if (!e || !out) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    Ctrl c;
    ISL_CUDA(e, cudaMemcpyAsync(&c, e->d_ctrl, sizeof(Ctrl), cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    e->st.placed = c.placed; e->st.freed = c.freed; e->st.no_capacity = c.allocs - c.placed; e->st.chain_steps = c.steps; e->st.chain_gpus_visited = c.visited; e->st.chain_jumps = c.jumps; e->st.scan_placed = c.scanned;
    e->st.spec_chunks = c.spec_cells; e->st.spec_rounds = c.spec_rounds; e->st.spec_sims = c.spec_sims;
    *out = e->st;
    return ISL_OK;
}

int isl_reset_stats(isl_engine* e) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    const uint64_t launches = e->st.kernel_launches;
    e->st = isl_stats{};
    e->st.kernel_launches = launches;      // launches are counted since creation
    ISL_CUDA(e, cudaMemsetAsync(&e->d_ctrl.get()->placed, 0, 8 * sizeof(unsigned long long), e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    return ISL_OK;
}

// ---- what-if / defragmentation queries (SURVEY 8f-4) -------------------------------------------------------------------
static int capacity_locked(isl_engine* e, uint64_t* cap) {
    ISL_CUDA(e, cudaMemsetAsync(e->d_cap, 0, ISL_MAX_PROFILES * sizeof(unsigned long long), e->stream));
    if (e->hi > e->lo) {
        k_capacity<<<std::min(ceil_div(e->hi - e->lo, 256), 296u), 256, 0, e->stream>>>(e->d_occ, e->d_gtab, e->d_capn, e->prof.n, e->lo, e->hi, e->d_cap);
        if (int rc = check_launch(e, "k_capacity")) return rc;
    }
    unsigned long long h[ISL_MAX_PROFILES];
    ISL_CUDA(e, cudaMemcpyAsync(h, e->d_cap, sizeof h, cudaMemcpyDeviceToHost, e->stream));
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) cap[p] = h[p];
    return ISL_OK;
}

int isl_capacity(isl_engine* e, uint64_t* cap) {
    if (!e || !cap) return ISL_EINVAL;
    Entry guard(e, Needs::ready);
    if (guard.rc) return guard.rc;
    return capacity_locked(e, cap);
}

int isl_what_if(isl_engine* e, uint32_t n, const isl_request* plan, isl_result* out, uint64_t* cap_before, uint64_t* cap_after) {
    if (!e || (n && (!plan || !out))) return ISL_EINVAL;
    Entry guard(e, Needs::ready, n);                // snapshot, plan, measurement and restore under ONE lock: nobody sees the hypothetical state
    if (guard.rc) return guard.rc;
    if (int rc = snapshot_occ(e)) return rc;
    int rc = ISL_OK;
    if (cap_before) rc = capacity_locked(e, cap_before);
    if (!rc && n) rc = place_batch_locked(e, n, plan, out);
    if (!rc && cap_after) rc = capacity_locked(e, cap_after);
    // the live state comes back whatever happened above
    const cudaError_t err = cudaMemcpyAsync(e->d_occ, e->d_occ_snap, e->occ_bytes, cudaMemcpyDeviceToDevice, e->stream);
    const cudaError_t err2 = cudaStreamSynchronize(e->stream);
    e->snap_G = 0;                                  // a caller's own snapshot (isl_snapshot_occupancy) does not survive a what-if
    if (!rc && (err != cudaSuccess || err2 != cudaSuccess)) { snprintf(e->cuda_err, sizeof(e->cuda_err), "isl_what_if restore: %s", cudaGetErrorString(err != cudaSuccess ? err : err2)); rc = ISL_ECUDA; }
    return rc;
}

// ---- causal window / pinned buffers / owner-gathered results --------------------------------------------------------------
int isl_set_causal_window(isl_engine* e, uint32_t window) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->window = window;
    return ISL_OK;
}

// debugging aid (not part of the boundary): the per-round stamps recorded under ISL_SPEC_DBG=chunk,stage; out: kSpecRounds x 8 uint64
int isl_debug_spec_rounds(isl_engine* e, uint64_t* out, uint32_t max_words) {
    if (!e || !out || !e->d_specdbg) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    ISL_CUDA(e, cudaStreamSynchronize(e->stream));
    ISL_CUDA(e, cudaMemcpy(out, e->d_specdbg, std::min<size_t>(max_words, kSpecRounds * 8) * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    return ISL_OK;
}

int isl_set_speculation(isl_engine* e, uint32_t mode) {
    if (!e || mode > ISL_SPEC_ON) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->spec_mode = mode;
    return ISL_OK;
}

int isl_set_ring_world(isl_engine* e, uint32_t world) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->ring_world = world;
    return ISL_OK;
}

void* isl_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}

void isl_host_free(void* p) { if (p) cudaFreeHost(p); }

void* isl_device_results(isl_engine* e) { return e ? e->d_res.get() : nullptr; }

int isl_ipc_results_handle(isl_engine* e, void* handle64) {
    if (!e || !handle64) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    return ipc_export(e, e->d_res, handle64);
}

int isl_ipc_connect_owner(isl_engine* e, const void* owner_handle64) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->d_owner_out.reset();
    if (owner_handle64) return ipc_open(e, owner_handle64, e->d_owner_out.out());
    return ISL_OK;
}

int isl_connect_owner_local(isl_engine* e, isl_engine* owner) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::nothing);
    if (guard.rc) return guard.rc;
    e->d_owner_out.borrow(owner ? owner->d_res.get() : nullptr);
    return ISL_OK;
}

// ---- open streams: the causal feed ----------------------------------------------------------------------------------------
// One persistent k_pipeline resolves batches that arrive WHILE it runs: isl_stream_submit copies a batch in and pre-passes it on the
// feed stream, the kernel's extra CTA writes its results into the caller's pinned buffer and raises a host-visible word, and
// isl_stream_wait returns as soon as that word is up — the caller composes batch b+1 (or b+k) from results it has already seen.
int isl_stream_open(isl_engine* e, uint32_t max_batches) {
    if (!e || max_batches == 0 || max_batches > kMaxStreamChunks) return ISL_EINVAL;
    Entry guard(e, Needs::ready);
    if (guard.rc) return guard.rc;
    if (request_major(e->cfg)) return ISL_EINVAL;
    // a tool that serialises kernels would starve a resident kernel that waits for kernels launched after it: refuse instead of hanging
    // until the device-side trap (callers fall back to isl_place_batch per batch)
    if (getenv("ISL_NO_FEED") || kernels_serialised()) {
        snprintf(e->cuda_err, sizeof(e->cuda_err), "isl_stream_open: kernel-serialising tool or ISL_NO_FEED set; open streams need concurrent kernels");
        return ISL_ESTATE;
    }
    auto& o = e->open;
    const uint32_t pc = e->pipe_chunk;
    if ((uint64_t)max_batches * pc > e->cfg.max_batch) return ISL_ERANGE;       // every batch owns a slot of the staging buffers
    // speculative rounds: the caller says (isl_set_causal_window) that it keeps at most 1..3 batches in flight, or asks for them outright;
    // their record memory stays within 1 GiB, is not shared with other ranks (route) and their stages leave room for the copier CTA and
    // the feed kernels
    PipePlan plan;
    if (int rc = plan_pipeline(e, std::max(2u, max_batches), (double)pc, true, false, e->window >= 1 && e->window <= 3,
                               !e->spec_shared && (uint64_t)max_batches * kSpecWordsPerChunk * 8ull <= (1ull << 30), true, &plan)) return rc;
    if (plan.n_seg + 1 + kFeedReserve > (uint32_t)e->max_coresident) return ISL_ERANGE;  // the feed kernels need SMs next to the resident pipeline
    o.plan = plan; o.max_batches = max_batches; o.submitted = 0; o.launched = false;
    o.q_stride = pc + kQPad * ISL_MAX_PROFILES; o.free_stride = (uint32_t)e->occ_bytes; o.tiles_per_batch = pc / kTile;
    if (int rc = grow_stream_buffers(e, max_batches, o.q_stride, max_batches * o.tiles_per_batch, max_batches, plan.n_seg, max_batches + 1, max_batches)) return rc;
    if ((uint64_t)max_batches * o.tiles_per_batch > ceil_div(e->cfg.max_batch, kTile) + 4096) return ISL_ERANGE;
    ISL_CUDA(e, o.h_done.reserve(max_batches));
    ISL_CUDA(e, o.h_chunks.reserve(max_batches));
    ISL_CUDA(e, o.h_tiles.reserve((size_t)max_batches * o.tiles_per_batch));
    memset(o.h_done, 0, (size_t)max_batches * sizeof(uint32_t));
    if (int rc = ensure_feed_stream(e)) return rc;
    if (int rc = next_epoch(e, &o.epoch)) return rc;
    if (plan.spec) if (int rc = prepare_spec(e, max_batches, o.epoch, e->stream)) return rc;
    // the feed stream starts behind whatever the engine's stream still holds
    ISL_CUDA(e, cudaEventRecord(e->ev_feed, e->stream));
    ISL_CUDA(e, cudaStreamWaitEvent(e->feed_stream, e->ev_feed, 0));
    ISL_CUDA(e, cudaMemsetAsync(e->d_done_cnt, 0, (size_t)max_batches * sizeof(uint32_t), e->feed_stream));
    ISL_CUDA(e, cudaMemsetAsync(e->d_ready, 0, (size_t)(max_batches + 1) * sizeof(uint32_t), e->feed_stream));
    ISL_CUDA(e, cudaMemsetAsync(e->d_free_acc, 0, (size_t)max_batches * o.free_stride, e->feed_stream));
    o.active = true;
    return ISL_OK;
}

int isl_stream_submit(isl_engine* e, uint32_t n, const isl_request* in, isl_result* out, uint32_t* ticket) {
    if (!e || n == 0 || !in || !out) return ISL_EINVAL;
    Entry guard(e, Needs::open_stream);
    if (guard.rc) return guard.rc;
    auto& o = e->open;
    if (o.submitted >= o.max_batches || n > e->pipe_chunk) return ISL_ERANGE;
    // the results are written by the running kernel: the destination must be mapped pinned host memory (isl_host_alloc, cudaHostAlloc,
    // cudaHostRegister)
    cudaPointerAttributes pa{};
    if (cudaPointerGetAttributes(&pa, out) != cudaSuccess || pa.type != cudaMemoryTypeHost || !pa.devicePointer) { cudaGetLastError(); return ISL_EINVAL; }
    const uint32_t b = o.submitted, pc = e->pipe_chunk, off = b * pc, tile0 = b * o.tiles_per_batch, n_tiles = ceil_div(n, kTile);
    const cudaStream_t pre = e->feed_stream;
    uint32_t chunk = b, tile = tile0;
    describe_batch(b, off, n, pc, o.h_chunks, chunk, o.h_tiles, tile);        // n <= pipe_chunk: one chunk
    o.h_chunks[b].host_out = static_cast<uint2*>(pa.devicePointer);
    ISL_CUDA(e, cudaMemcpyAsync(e->d_chunks + b, o.h_chunks + b, sizeof(ChunkDesc), cudaMemcpyHostToDevice, pre));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_tiles + tile0, o.h_tiles + tile0, (size_t)n_tiles * sizeof(TileDesc), cudaMemcpyHostToDevice, pre));
    ISL_CUDA(e, cudaMemcpyAsync(e->d_req + off, in, (size_t)n * sizeof(isl_request), cudaMemcpyHostToDevice, pre));
    k_prepare<<<n_tiles, kTileThreads, 0, pre>>>(0, e->d_req, e->d_res, reinterpret_cast<uint32_t*>(e->d_occ.get()), e->G, e->lo, e->hi, e->prof,
                                                 e->d_tile_counts, e->d_ctrl, e->d_tiles, e->d_free_acc, o.free_stride / 4, tile0);
    if (int rc = check_launch(e, "k_prepare")) return rc;
    k_partition<<<n_tiles, kTileThreads, 0, pre>>>(0, e->d_req, e->prof.n, e->d_tile_counts, 0, e->cand_profiles, e->d_qall, e->d_cctl,
                                                   e->d_tiles, o.q_stride, tile0);
    if (int rc = check_launch(e, "k_partition")) return rc;
    k_set_flag<<<1, 1, 0, pre>>>(e->d_ready + b, o.epoch);
    if (int rc = check_launch(e, "k_set_flag")) return rc;
    if (!o.launched) {          // the persistent pipeline starts behind the first batch's tables
        ISL_CUDA(e, cudaEventRecord(e->ev_feed, pre));
        ISL_CUDA(e, cudaStreamWaitEvent(e->stream, e->ev_feed, 0));
        PipeArgs args = pipe_args(e, o.plan, o.max_batches, o.epoch, o.q_stride, e->d_res);
        args.ready = e->d_ready; args.done_cnt = e->d_done_cnt; args.copier = 1; args.open = 1; args.host_done = o.h_done.dev();
        args.wait_ns = std::max(kOpenWaitNs, e->wait_ns);
        if (int rc = start_pipeline(e, args)) return rc == ISL_ESTATE ? ISL_ERANGE : rc;
        o.launched = true;
    }
    if (ticket) *ticket = b;
    ++o.submitted;
    ++e->st.batches; e->st.requests += n;
    return ISL_OK;
}

int isl_stream_wait(isl_engine* e, uint32_t ticket) {
    if (!e) return ISL_EINVAL;
    auto& o = e->open;
    if (!o.active || ticket >= o.submitted) return ISL_ESTATE;
    // no lock: only reads a word the device raises; other threads may keep submitting
    volatile uint32_t* flag = o.h_done + ticket;
    const uint32_t epoch = o.epoch;
    uint64_t spins = 0;
    while (*flag != epoch) {
        if ((++spins & 0xFFFFu) == 0) {                 // now and then: did the pipeline die (a trap, an earlier launch error)?
            DeviceGuard guard(e->device);
            const cudaError_t err = cudaStreamQuery(e->stream);
            if (err != cudaSuccess && err != cudaErrorNotReady) { snprintf(e->cuda_err, sizeof(e->cuda_err), "isl_stream_wait: %s", cudaGetErrorString(err)); return ISL_ECUDA; }
            if (err == cudaSuccess && *flag != epoch) { snprintf(e->cuda_err, sizeof(e->cuda_err), "isl_stream_wait: pipeline ended before batch %u", ticket); return ISL_ECUDA; }
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return ISL_OK;
}

int isl_stream_close(isl_engine* e) {
    if (!e) return ISL_EINVAL;
    Entry guard(e, Needs::open_stream);
    if (guard.rc) return guard.rc;
    auto& o = e->open;
    int rc = ISL_OK;
    if (o.launched) {
        if (o.submitted < o.max_batches) {
            k_set_flag<<<1, 1, 0, e->feed_stream>>>(e->d_ready + o.submitted, ~o.epoch);     // 'closed': the kernel leaves its chunk loop
            rc = check_launch(e, "k_set_flag");
        }
        cudaError_t err = cudaStreamSynchronize(e->feed_stream);
        if (err == cudaSuccess) err = cudaStreamSynchronize(e->stream);
        if (err != cudaSuccess) { snprintf(e->cuda_err, sizeof(e->cuda_err), "isl_stream_close: %s", cudaGetErrorString(err)); rc = ISL_ECUDA; }
    } else {
        cudaStreamSynchronize(e->feed_stream);
    }
    o.active = false; o.launched = false;
    return rc;
}

}  // extern "C"
