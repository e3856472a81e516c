// isl_kernels.cuh — sm_90a kernels of the MIG-slot placement engine.
//
// Replaces, for a whole batch of pending pods at once, the reference's per-pod scan
//   Reconcile node loop            internal/controller/instaslice_controller.go:190
//   findDeviceForASlice GPU loop   :240-262
//   getStartIndexFromPreparedState :303-384
// Pure integer / bitmask work: no tensor cores, nothing to reshape into a GEMM.
//
// Pipeline per batch (DESIGN.md "Kernels"):
//   k_prepare            frees (atomicAnd on packed occupancy words), default results, per-tile
//                        per-profile histogram of the ALLOC requests
//   per chunk of <= 65536 requests:
//     k_partition        stable P-way partition of the chunk's ALLOC requests into per-profile queues
//     k_sweep_count/_scatter   vectorised sweep over the occupancy bytes: feasibility bitmask via a
//                        256-entry shared-memory table, ordered compaction of the candidate GPUs
//     k_chain<K>         exact first-fit commit: GPU-major stream filtering with one lane per
//                        (profile, start) candidate and a warp min-reduction per accepted placement
#pragma once

#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/islplace.h"

namespace isl {

constexpr uint32_t kChunk = 65536;         // requests per commit chunk: in-chunk request index fits 16 bits
constexpr uint32_t kTile = 1024;           // requests per partition tile (256 threads x 4 rounds)
constexpr uint32_t kTileThreads = 256;
constexpr uint32_t kTilesPerChunk = kChunk / kTile;
constexpr uint32_t kQPad = 32;             // per-profile queue segments start on 32-entry boundaries
constexpr uint32_t kQCap = kChunk + kQPad * ISL_MAX_PROFILES;
constexpr uint32_t kSweepThreads = 256;
constexpr uint32_t kSweepPerThread = 16;   // one 16-byte vector load = 16 GPUs
constexpr uint32_t kSweepBlock = kSweepThreads * kSweepPerThread;   // 4096 GPUs per CTA
constexpr uint32_t kSkip = 0xFFu;          // partition key of a request that is not a valid ALLOC
constexpr uint32_t kInf = 0xFFFFFFFFu;
constexpr uint32_t kMaxCand = ISL_MAX_PROFILES * ISL_MAX_STARTS;   // 128 (profile,start) candidates
constexpr uint32_t kChainThreads = 256;
constexpr uint32_t kMaxTables = ISL_MAX_TABLES;   // per-node profile tables (heterogeneous clusters)

// The chain's occupancy word is 16 bits: the busy slices in the low byte and, in the high byte, every table bit set EXCEPT
// the one of the table the GPU's node publishes.  A candidate of table t carries bit (8 + t) in its mask, so `(occ16 & mask) == 0`
// holds only on GPUs of its own table — no extra instruction per decision.
// The decision loop's tuning choices (DESIGN.md 4.1) are plain constants; a variant is built by editing the constant.
// true for every lane of warp 0 and only there.  The predicate comes out of a redux (a uniform register): ptxas then knows the warp is
// converged and drops the BRA.DIV / UMOV guard in front of every redux of the loop.
__device__ __forceinline__ bool is_chain_warp(uint32_t warp) { return __reduce_or_sync(0xFFFFFFFFu, warp) == 0; }

__host__ __device__ inline uint32_t table_tag(uint32_t table) { return ((~(1u << table)) & 0xFFu) << 8; }

struct DevProfiles {            // kernel parameter (by value)
    uint32_t n;
    uint32_t quirks;
    isl_profile rows[ISL_MAX_PROFILES];
    uint32_t flip;              // ISL_POLICY_RIGHT_TO_LEFT: G (the inventory is stored in REVERSE canonical order), else 0
};

// ISL_POLICY_RIGHT_TO_LEFT walks the GPUs in descending canonical order.  The engine stores such an inventory reversed (internal index
// i = G - 1 - canonical) so that every scan stays an ascending sweep; only the two edges translate: the GPU a FREE names, and the GPU a
// PLACED record reports.
__host__ __device__ inline uint32_t flip_gpu(uint32_t g, uint32_t flip) { return flip ? flip - 1u - g : g; }

// One (profile, start) candidate of the chain: bits  [3:0] profile | [6:4] order in the row |
// [10:7] start | [14:11] size | [23:16] slot mask | [26:24] table | [31] valid
struct CandTab {                // kernel parameter (by value): slot k of lane l is desc[k][l]
    uint32_t desc[4][32];
};

struct Ctrl {                   // device-resident control block, rewritten per chunk
    uint32_t qoff[ISL_MAX_PROFILES + 1];   // queue segment offsets (entries) inside the chunk's queue buffer
    uint32_t qcnt[ISL_MAX_PROFILES];       // requests of profile p in this chunk
    uint32_t active;                       // profiles with requests in this chunk AND >= 1 valid candidate
    uint32_t n_cand;                       // candidate GPUs found by the sweep
    uint32_t n_log;                        // decisions logged by the chain of this chunk
    unsigned long long placed, freed, bad, steps, visited, allocs, jumps, scanned;
    unsigned long long spec_sims, spec_rounds, spec_cells;   // speculative rounds: segment simulations run (all stages), rounds until the last stage was certified summed over chunks, chunks
};

// The batch counters of a kernel that commits its own placements, one decision step per placed request.
__device__ __forceinline__ void count_placed(Ctrl* ctrl, uint32_t placed) {
    atomicAdd(&ctrl->placed, (unsigned long long)placed);
    atomicAdd(&ctrl->steps, (unsigned long long)placed);
}

// Slot mask of `size` slices from slice `start`, cut to the GPU's byte.
__host__ __device__ inline uint32_t slice_span(uint32_t start, uint32_t size) { return (((1u << size) - 1u) << start) & 0xFFu; }

// The one rule both the device table and the chain candidates come from: slot mask of placing a
// `size`-slice profile at start v, or 0 when getStartIndexFromPreparedState can never return v
//   size 1            -> only busy[v] is tested (:346-349)
//   size 2/4/8        -> needs v+size < 8 (strict, Q1) and all slots free (:350-378)
//   any other size    -> never placed under Q2; with the quirk off, any size 2..8 with v+size <= 8
__host__ __device__ inline uint32_t candidate_mask(uint32_t size, uint32_t v, uint32_t quirks) {
    if (v >= ISL_SLOTS || size == 0 || size > ISL_SLOTS) return 0;
    if (size == 1) return 1u << v;
    const bool pow2_only = quirks & ISL_QUIRK_POW2_ONLY;
    if (pow2_only && !(size == 2 || size == 4 || size == 8)) return 0;
    const bool strict = quirks & ISL_QUIRK_STRICT_BOUND;
    if (strict ? !(v + size < ISL_SLOTS) : !(v + size <= ISL_SLOTS)) return 0;
    return slice_span(v, size);
}

// ---------------------------------------------------------------------------------------------
// Device table: lut[p][occ] = first legal start of profile p on a GPU with occupancy byte occ
// (or 9), feas[occ] = bitmask of profiles that have a legal start.  256 threads, one per byte.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_build_lut(DevProfiles prof, uint32_t table, uint8_t* __restrict__ lut, uint16_t* __restrict__ feas,
                                                   uint8_t* __restrict__ capn, uint32_t* __restrict__ seq) {
    lut += (size_t)table * ISL_MAX_PROFILES * 256; feas += (size_t)table * 256;        // lut[table][profile][occ], feas[table][occ]
    capn += (size_t)table * ISL_MAX_PROFILES * 256; seq += (size_t)table * ISL_MAX_PROFILES * 256;
    const uint32_t occ = threadIdx.x;
    uint32_t fmask = 0;
    for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) {
        uint32_t found = ISL_START_NONE;
        if (p < prof.n) {
            const isl_profile& row = prof.rows[p];
            for (uint32_t k = 0; k < row.n_starts; ++k) {                        // CRD order (:344)
                const uint32_t m = candidate_mask(row.size, row.starts[k], prof.quirks);
                if (m != 0 && (occ & m) == 0) { found = row.starts[k]; break; }
            }
        }
        lut[p * 256 + occ] = (uint8_t)found;
        if (found != ISL_START_NONE) fmask |= 1u << p;
        // how many requests of this profile the GPU takes IN A ROW from this occupancy, and at which starts (4 bits each):
        // the single-profile scan commit (k_sweep_* in scan mode) places whole GPUs at once from these two tables
        uint32_t o = occ, cnt = 0, packed = 0;
        if (p < prof.n) {
            const isl_profile& row = prof.rows[p];
            while (cnt < 8) {
                uint32_t st = ISL_START_NONE, mk = 0;
                for (uint32_t k = 0; k < row.n_starts; ++k) {
                    const uint32_t m = candidate_mask(row.size, row.starts[k], prof.quirks);
                    if (m != 0 && (o & m) == 0) { st = row.starts[k]; mk = m; break; }
                }
                if (st == ISL_START_NONE) break;
                packed |= st << (4 * cnt); o |= mk; ++cnt;
            }
        }
        capn[p * 256 + occ] = (uint8_t)cnt;
        seq[p * 256 + occ] = packed;
    }
    feas[occ] = (uint16_t)fmask;
}

__global__ void k_eval_starts(const uint8_t* __restrict__ lut, uint32_t profile, uint32_t n,
                              const uint8_t* __restrict__ occ, uint8_t* __restrict__ out) {
    __shared__ uint8_t s_lut[256];
    if (threadIdx.x < 256) s_lut[threadIdx.x] = lut[profile * 256 + threadIdx.x];
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = s_lut[occ[i]];
}

// A release of `size` slices from `start` on canonical GPU `gpu`: false for a malformed span (BAD_SPAN).  Otherwise `gi` is where the
// engine keeps that GPU and `span` the slot mask shifted into the GPU's byte of its packed occupancy word, or 0 when gi is outside [lo, hi).
__device__ __forceinline__ bool free_span(uint32_t gpu, uint32_t start, uint32_t size, uint32_t G, uint32_t lo, uint32_t hi, uint32_t flip,
                                          uint32_t& gi, uint32_t& span) {
    span = 0;
    if (gpu >= G || size == 0 || start + size > ISL_SLOTS) return false;
    gi = flip_gpu(gpu, flip);
    if (gi >= lo && gi < hi) span = slice_span(start, size) << ((gi & 3u) * 8u);      // start + size <= 8: the cut changes nothing
    return true;
}

__global__ void k_free_spans(uint32_t n, const isl_span* __restrict__ spans, uint32_t* __restrict__ occ32,
                             uint32_t G, uint32_t lo, uint32_t hi, Ctrl* ctrl, uint32_t flip) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const isl_span s = spans[i];
    uint32_t gi, span;
    if (!free_span(s.gpu, s.start, s.size, G, lo, hi, flip, gi, span)) { atomicAdd(&ctrl->bad, 1ull); return; }
    if (!span) return;
    atomicAnd(&occ32[gi >> 2], ~span);
    atomicAdd(&ctrl->freed, 1ull);
}

// ---------------------------------------------------------------------------------------------
// k_prepare: one pass over the request stream (8 B coalesced loads, 8 B coalesced stores).
//   FREE  -> clear the span in the packed occupancy word, result FREED / BAD_SPAN
//   ALLOC -> default result (gpu NONE, start 9, NO_CAPACITY); the chain overwrites what it places
//   per-tile histogram of ALLOC requests by profile (warp match + one shared atomic per group)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint2 pack_result(uint32_t gpu, uint32_t start, uint32_t size, uint32_t status) {
    return make_uint2(gpu, start | (size << 8) | (status << 16));
}

// The per-request step every pre-pass shares (k_prepare, k_small phase A, k_few): decodes the request, writes its default record
// (ALLOC: NO_CAPACITY or BAD_PROFILE; FREE: FREED or BAD_SPAN; anything else: NOOP) and returns its partition key (the profile of a valid
// ALLOC, else kSkip).  For a valid FREE inside [lo, hi), `gi` and `span` (non-zero) say what to release; the caller applies it.
__device__ __forceinline__ uint32_t prepare_request(uint2 rq, uint2& out, const DevProfiles& prof, uint32_t G, uint32_t lo, uint32_t hi,
                                                    uint32_t& gi, uint32_t& span) {
    const uint32_t handle = rq.x, profile = rq.y & 0xFFu, op = (rq.y >> 8) & 0xFFu, start = (rq.y >> 16) & 0xFFu, size = rq.y >> 24;
    span = 0;
    if (op == ISL_OP_ALLOC) {
        if (profile < prof.n) { out = pack_result(ISL_GPU_NONE, ISL_START_NONE, prof.rows[profile].size, ISL_ST_NO_CAPACITY); return profile; }
        out = pack_result(ISL_GPU_NONE, ISL_START_NONE, 0, ISL_ST_BAD_PROFILE);
    } else if (op == ISL_OP_FREE) {
        const bool ok = free_span(handle, start, size, G, lo, hi, prof.flip, gi, span);
        out = pack_result(handle, start, size, ok ? ISL_ST_FREED : ISL_ST_BAD_SPAN);
    } else out = pack_result(ISL_GPU_NONE, ISL_START_NONE, 0, ISL_ST_NOOP);
    return kSkip;
}

// One logged decision of the chain (key, candidate index): the PLACED record of its request, and the slot mask ORed into the packed
// occupancy word.  Distinct decisions on one GPU have disjoint masks (the chain only accepts free masks): the atomic only serialises
// neighbours that share a word.  `cand` may have been written by the calling kernel, hence the L2 load.
__device__ __forceinline__ void commit_decision(uint2 e, const uint32_t* cand, uint32_t* occ32, uint2* out, uint32_t flip) {
    const uint32_t g = __ldcg(cand + e.y) >> 8, mask = e.x & 0xFFu, t = (e.x >> 15) & 0xFFFFu;
    out[t] = pack_result(flip_gpu(g, flip), __ffs(mask) - 1, __popc(mask), ISL_ST_PLACED);
    atomicOr(&occ32[g >> 2], mask << ((g & 3u) * 8u));
}

// One tile of 1024 requests of a stream: which batch / pipeline chunk it belongs to (host-built table, one launch
// of k_prepare and one of k_partition cover every batch and chunk of a stream call).
struct TileDesc {
    uint32_t batch_off, batch_n, batch, batch_first_tile;      // batch: request offset in the stream, size, index, first global tile
    uint32_t chunk, chunk_first_tile, chunk_tiles, chunk_off;  // chunk: index, first global tile, tiles, request offset in the stream
    uint32_t chunk_n, pad0, pad1, pad2;
};

__global__ void __launch_bounds__(kTileThreads) k_prepare(uint32_t n, const uint2* __restrict__ in, uint2* __restrict__ out,
                                                           uint32_t* __restrict__ occ32, uint32_t G, uint32_t lo, uint32_t hi,
                                                           DevProfiles prof, uint32_t* __restrict__ tile_counts, Ctrl* ctrl,
                                                           const TileDesc* __restrict__ descs, uint32_t* __restrict__ free_acc, uint32_t free_stride,
                                                           uint32_t tile_base) {
    // descs != nullptr (stream mode): the tile's batch comes from the table, and FREEs are not applied here but ORed
    // into the batch's free-mask array (one byte per GPU); the segment pipeline clears them in batch order inside the
    // segment that owns the GPU.  tile_base: first global tile of this launch (a stream may be fed batch by batch).
    const uint32_t bid = blockIdx.x + tile_base;
    uint32_t tile = bid;
    if (descs) {
        const TileDesc d = descs[bid];
        n = d.batch_n; in += d.batch_off; out += d.batch_off; tile = bid - d.batch_first_tile;
        free_acc += (size_t)d.batch * free_stride;
    }
    __shared__ uint32_t s_cnt[ISL_MAX_PROFILES];
    __shared__ uint32_t s_freed;
    if (threadIdx.x < ISL_MAX_PROFILES) s_cnt[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_freed = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31u;
#pragma unroll
    for (uint32_t r = 0; r < kTile / kTileThreads; ++r) {
        const uint32_t i = tile * kTile + r * kTileThreads + threadIdx.x;
        uint32_t key = kSkip;
        if (i < n) {
            uint32_t gi, span;
            key = prepare_request(in[i], out[i], prof, G, lo, hi, gi, span);
            if (span) {
                if (descs) atomicOr(&free_acc[gi >> 2], span);
                else atomicAnd(&occ32[gi >> 2], ~span);
                atomicAdd(&s_freed, 1u);
            }
        }
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key);
        if (key != kSkip && lane == (uint32_t)(__ffs(peers) - 1)) atomicAdd(&s_cnt[key], (uint32_t)__popc(peers));
    }
    __syncthreads();
    if (threadIdx.x < ISL_MAX_PROFILES) tile_counts[bid * ISL_MAX_PROFILES + threadIdx.x] = s_cnt[threadIdx.x];
    if (threadIdx.x == 0) {
        if (s_freed) atomicAdd(&ctrl->freed, (unsigned long long)s_freed);
        uint32_t allocs = 0;
        for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) allocs += s_cnt[p];
        if (allocs) atomicAdd(&ctrl->allocs, (unsigned long long)allocs);
    }
}

// ---------------------------------------------------------------------------------------------
// k_partition: stable P-way partition of one chunk's ALLOC requests.  Queue p receives the
// in-chunk indices (16 bit) of the requests for profile p, in request order.
// grid = tiles of the chunk; every CTA re-derives the chunk-wide offsets from tile_counts
// (<= 64 tiles x 16 counters), so no inter-CTA communication is needed.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTileThreads) k_partition(uint32_t n_chunk, const uint2* __restrict__ in_chunk, uint32_t n_profiles,
                                                             const uint32_t* __restrict__ tile_counts_chunk, uint32_t n_tiles,
                                                             uint32_t cand_profiles, uint16_t* __restrict__ q, Ctrl* ctrl,
                                                             const TileDesc* __restrict__ descs, uint32_t q_stride, uint32_t tile_base) {
    // descs != nullptr (stream mode): in_chunk / tile_counts_chunk / q / ctrl are the bases of the whole stream and
    // the tile's chunk comes from the table.
    const uint32_t bid = blockIdx.x + tile_base;
    uint32_t tile = bid;
    if (descs) {
        const TileDesc d = descs[bid];
        n_chunk = d.chunk_n; in_chunk += d.chunk_off; tile_counts_chunk += (size_t)d.chunk_first_tile * ISL_MAX_PROFILES;
        n_tiles = d.chunk_tiles; tile = bid - d.chunk_first_tile; q += (size_t)d.chunk * q_stride; ctrl += d.chunk;
    }
    __shared__ uint32_t s_part[16][ISL_MAX_PROFILES][2];   // [j][p][0]=total, [1]=prefix before this tile
    __shared__ uint32_t s_base[ISL_MAX_PROFILES];
    __shared__ uint32_t s_seg[32][ISL_MAX_PROFILES];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    {   // chunk-wide per-profile totals and the prefix of the tiles before this one
        const uint32_t p = tid & 15u, j = tid >> 4;
        uint32_t tot = 0, pre = 0;
        for (uint32_t t = j; t < n_tiles; t += 16) {
            const uint32_t c = tile_counts_chunk[t * ISL_MAX_PROFILES + p];
            tot += c;
            if (t < tile) pre += c;
        }
        s_part[j][p][0] = tot; s_part[j][p][1] = pre;
    }
    for (uint32_t k = tid; k < 32 * ISL_MAX_PROFILES; k += kTileThreads) (&s_seg[0][0])[k] = 0;
    __syncthreads();
    if (tid == 0) {
        uint32_t off = 0, active = 0;
        for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) {
            uint32_t tot = 0, pre = 0;
            for (uint32_t j = 0; j < 16; ++j) { tot += s_part[j][p][0]; pre += s_part[j][p][1]; }
            s_base[p] = off + pre;
            if (tile == 0) {
                ctrl->qoff[p] = off; ctrl->qcnt[p] = tot;
                if (tot && ((cand_profiles >> p) & 1u)) active |= 1u << p;
            }
            off += (tot + kQPad - 1) & ~(kQPad - 1);
        }
        if (tile == 0) { ctrl->qoff[ISL_MAX_PROFILES] = off; ctrl->active = active; ctrl->n_cand = 0; }
    }
    uint32_t key[4], rank[4];
#pragma unroll
    for (uint32_t r = 0; r < 4; ++r) {
        const uint32_t i = tile * kTile + r * kTileThreads + tid;
        key[r] = kSkip;
        if (i < n_chunk) {
            const uint32_t w = in_chunk[i].y;
            const uint32_t profile = w & 0xFFu, op = (w >> 8) & 0xFFu;
            if (op == ISL_OP_ALLOC && profile < n_profiles) key[r] = profile;
        }
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key[r]);
        rank[r] = __popc(peers & ((1u << lane) - 1u));
        if (key[r] != kSkip && lane == (uint32_t)(__ffs(peers) - 1)) s_seg[r * 8 + warp][key[r]] = __popc(peers);
    }
    __syncthreads();
    if (tid < ISL_MAX_PROFILES) {           // exclusive scan over the 32 (round, warp) segments, in request order
        uint32_t run = 0;
        for (uint32_t s = 0; s < 32; ++s) { const uint32_t c = s_seg[s][tid]; s_seg[s][tid] = run; run += c; }
    }
    __syncthreads();
#pragma unroll
    for (uint32_t r = 0; r < 4; ++r) {
        if (key[r] == kSkip) continue;
        const uint32_t i = tile * kTile + r * kTileThreads + tid;
        q[s_base[key[r]] + s_seg[r * 8 + warp][key[r]] + rank[r]] = (uint16_t)i;
    }
}

// one word, stream-ordered: "the pre-pass of this batch is complete" for a segment pipeline that is already running
__global__ void k_set_flag(uint32_t* flag, uint32_t value) {
    __threadfence();
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
}

// ---------------------------------------------------------------------------------------------
// Sweep: every thread loads 16 occupancy bytes with one 128-bit read-only load, looks each byte
// up in the 256-entry feasibility table staged in shared memory, and keeps the GPUs on which at
// least one profile that is pending in this chunk has a legal start.  Two passes (count, then
// ordered scatter) keep the candidate list in canonical GPU order without inter-CTA spinning.
// Candidate record = (gpu << 8) | occupancy byte.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_nc_v4(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// byte j (0..15) of a 16-byte vector of occupancy or table bytes: the byte of the vector's j-th GPU
__device__ __forceinline__ uint32_t byte16(const uint32_t (&w)[4], uint32_t j) { return (w[j >> 2] >> ((j & 3u) * 8u)) & 0xFFu; }
__device__ __forceinline__ uint32_t byte16(const uint4 v, uint32_t j) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    return byte16(w, j);
}

__device__ __forceinline__ uint32_t sweep_mask16(const uint4 v, const uint4 tv, const uint16_t* s_feas, uint32_t active, uint32_t g0, uint32_t lo, uint32_t hi) {
    uint32_t mask = 0;
#pragma unroll
    for (uint32_t j = 0; j < 16; ++j) {
        const uint32_t o = byte16(v, j), t = byte16(tv, j) & (kMaxTables - 1);
        const uint32_t g = g0 + j;
        if ((s_feas[t * 256 + o] & active) && g >= lo && g < hi) mask |= 1u << j;
    }
    return mask;
}

// Scan mode (exactly ONE placeable profile in the chunk, e.g. a burst of replicas of one Deployment): there is nothing
// to interleave, GPU g simply takes the next capn[occ_g] requests of the queue.  The two sweep passes then compute the
// device-wide exclusive scan of those capacities and commit results and occupancy directly — fully parallel, no chain.
__device__ __forceinline__ uint32_t scan_capacity16(const uint4 v, const uint4 tv, const uint8_t* __restrict__ capn, uint32_t p, uint32_t g0, uint32_t lo, uint32_t hi) {
    uint32_t c = 0;
#pragma unroll
    for (uint32_t j = 0; j < 16; ++j) {
        const uint32_t o = byte16(v, j), t = byte16(tv, j) & (kMaxTables - 1);
        const uint32_t g = g0 + j;
        if (g >= lo && g < hi) c += capn[(t * ISL_MAX_PROFILES + p) * 256 + o];
    }
    return c;
}

// Ordered compaction of the GPUs a 16-GPU sweep found feasible (`mask`), from position `off` on.  Returns the position after the last.
__device__ __forceinline__ uint32_t emit_candidates(uint32_t mask, const uint4 v, const uint4 tv, uint32_t g0, uint32_t off,
                                                    uint32_t* __restrict__ cand, uint16_t* __restrict__ cand_o16) {
    while (mask) {
        const uint32_t j = __ffs(mask) - 1; mask &= mask - 1;
        const uint32_t o = byte16(v, j), t = byte16(tv, j) & (kMaxTables - 1);
        cand_o16[off] = (uint16_t)(o | table_tag(t));          // what the chain needs: occupancy + table tag
        cand[off++] = ((g0 + j) << 8) | o;                       // what the commit needs: the GPU
    }
    return off;
}

__global__ void __launch_bounds__(kSweepThreads) k_sweep_count(const uint4* __restrict__ occ16, const uint4* __restrict__ gtab16, const uint16_t* __restrict__ feas,
                                                                uint32_t first_block, uint32_t lo, uint32_t hi,
                                                                const Ctrl* __restrict__ ctrl, uint32_t* __restrict__ counts, const uint8_t* __restrict__ capn) {
    __shared__ uint16_t s_feas[kMaxTables * 256];
    __shared__ uint32_t s_warp[kSweepThreads / 32];
    for (uint32_t i = threadIdx.x; i < kMaxTables * 256; i += kSweepThreads) s_feas[i] = feas[i];
    __syncthreads();
    const uint32_t active = ctrl->active;
    const uint32_t g0 = (first_block + blockIdx.x) * kSweepBlock + threadIdx.x * kSweepPerThread;
    uint32_t c = 0;
    if (active && g0 < hi && g0 + kSweepPerThread > lo) {
        const uint4 v = ld_nc_v4(&occ16[g0 >> 4]), tv = ld_nc_v4(&gtab16[g0 >> 4]);
        c = __popc(active) == 1 ? scan_capacity16(v, tv, capn, __ffs(active) - 1, g0, lo, hi) : __popc(sweep_mask16(v, tv, s_feas, active, g0, lo, hi));
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, d);
    if ((threadIdx.x & 31u) == 0) s_warp[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (uint32_t w = 0; w < kSweepThreads / 32; ++w) t += s_warp[w];
        counts[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(kSweepThreads) k_sweep_scatter(const uint4* __restrict__ occ16, const uint4* __restrict__ gtab16, const uint16_t* __restrict__ feas,
                                                                  uint32_t first_block, uint32_t lo, uint32_t hi, Ctrl* ctrl,
                                                                  const uint32_t* __restrict__ counts, uint32_t* __restrict__ cand,
                                                                  uint16_t* __restrict__ cand_o16, const uint8_t* __restrict__ capn, const uint32_t* __restrict__ seq,
                                                                  const uint16_t* __restrict__ q, uint8_t* __restrict__ occ8, uint2* __restrict__ out_chunk,
                                                                  const uint32_t* __restrict__ heads_in, uint32_t* __restrict__ heads_out, const uint8_t* __restrict__ sizes, uint32_t flip) {
    __shared__ uint16_t s_feas[kMaxTables * 256];
    __shared__ uint32_t s_warp[kSweepThreads / 32];
    __shared__ uint32_t s_red[kSweepThreads / 32];
    __shared__ uint32_t s_base;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    for (uint32_t i = tid; i < kMaxTables * 256; i += kSweepThreads) s_feas[i] = feas[i];
    // base = number of candidates in the CTAs before this one (and the grand total for the last CTA)
    uint32_t pre = 0;
    for (uint32_t b = tid; b < blockIdx.x; b += kSweepThreads) pre += counts[b];
#pragma unroll
    for (int d = 16; d; d >>= 1) pre += __shfl_xor_sync(0xFFFFFFFFu, pre, d);
    if (lane == 0) s_red[warp] = pre;
    __syncthreads();
    if (tid == 0) { uint32_t t = 0; for (uint32_t w = 0; w < kSweepThreads / 32; ++w) t += s_red[w]; s_base = t; }
    const uint32_t active = ctrl->active;
    const uint32_t g0 = (first_block + blockIdx.x) * kSweepBlock + tid * kSweepPerThread;
    uint4 v = make_uint4(0, 0, 0, 0), tv = make_uint4(0, 0, 0, 0);
    uint32_t mask = 0;
    const bool scan_mode = __popc(active) == 1;
    const uint32_t sp = scan_mode ? __ffs(active) - 1 : 0u;
    uint32_t cap_sum = 0;
    if (active && g0 < hi && g0 + kSweepPerThread > lo) {
        v = ld_nc_v4(&occ16[g0 >> 4]); tv = ld_nc_v4(&gtab16[g0 >> 4]);
        if (scan_mode) cap_sum = scan_capacity16(v, tv, capn, sp, g0, lo, hi);
        else mask = sweep_mask16(v, tv, s_feas, active, g0, lo, hi);
    }
    const uint32_t c = scan_mode ? cap_sum : __popc(mask);
    uint32_t incl = c;                                  // inclusive warp scan of the per-thread counts
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += t; }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t off = s_base + incl - c;
    for (uint32_t w = 0; w < warp; ++w) off += s_warp[w];
    if (scan_mode) {        // `off` is the exclusive scan of the capacities = queue position this thread's first GPU starts at
        const uint32_t h0 = heads_in ? heads_in[sp] : 0u, n_p = ctrl->qcnt[sp];
        const uint16_t* qp = q + ctrl->qoff[sp];
        uint32_t pos = h0 + off;
        if (cap_sum && pos < n_p) {
#pragma unroll 1
            for (uint32_t j = 0; j < 16 && pos < n_p; ++j) {
                const uint32_t g = g0 + j;
                if (g < lo || g >= hi) continue;
                const uint32_t o = byte16(v, j), t = byte16(tv, j) & (kMaxTables - 1);
                const uint32_t row = (t * ISL_MAX_PROFILES + sp) * 256 + o;
                const uint32_t cg = capn[row], size = sizes[t * ISL_MAX_PROFILES + sp];
                if (!cg) continue;
                uint32_t starts = seq[row], o2 = o;
                for (uint32_t k = 0; k < cg && pos < n_p; ++k, ++pos) {
                    const uint32_t st = (starts >> (4 * k)) & 15u;
                    out_chunk[qp[pos]] = pack_result(flip_gpu(g, flip), st, size, ISL_ST_PLACED);
                    o2 |= slice_span(st, size);
                }
                occ8[g] = (uint8_t)o2;
            }
        }
        if (blockIdx.x == gridDim.x - 1 && tid == kSweepThreads - 1) {      // `off + cap_sum` = total capacity of the range
            const uint32_t total = off + cap_sum, left = n_p > h0 ? n_p - h0 : 0u, placed = min(total, left);
            ctrl->n_cand = 0; ctrl->n_log = 0;                              // the chain and k_commit have nothing to do
            if (heads_out) heads_out[sp] = h0 + placed;
            if (placed) { atomicAdd(&ctrl->placed, (unsigned long long)placed); atomicAdd(&ctrl->scanned, (unsigned long long)placed); }
        }
        return;
    }
    off = emit_candidates(mask, v, tv, g0, off, cand, cand_o16);
    if (blockIdx.x == gridDim.x - 1 && tid == kSweepThreads - 1) ctrl->n_cand = off;
}

// ---------------------------------------------------------------------------------------------
// k_chain<K>: the exact commit decision chain.
//
// First-fit in canonical GPU order is GPU-major stream filtering: GPU g accepts, in request
// order, a prefix of each profile's remaining queue (occupancy only grows inside an alloc phase, so
// a profile that stopped fitting on g never fits again).  The state between GPUs is one queue head
// per profile.  The chain is a latency-bound sequential recurrence, so ONE warp walks the candidate
// GPUs and does nothing but decide; lane l owns up to K (profile, start) candidates with their slot
// masks in registers.  One warp min-reduction per accepted placement answers "which pending
// request is next and where does it start", looking at the current candidate GPU and the one after
// it at once:
//     key = sel << 31 | t << 15 | profile << 11 | order << 8 | mask
//       sel  0 = the candidate's mask is free on the current GPU, 1 = only on the next GPU
//       t    in-chunk index of the next pending request of the candidate's profile
//     m = warp-min(key):  lowest GPU first, then earliest request, then first legal start in row order
//     occupancy |= m & 0xFF; the lanes of the winning profile pop their queue head.
// Every decision is appended to a log (8 B: m, candidate index); k_commit turns the log into result
// records and occupancy updates with full parallelism afterwards.
// m == INF means neither GPU can take anything: a ballot over the feasibility table jumps straight to
// the next candidate GPU on which a profile that still has pending requests fits.
// The queues (16-bit in-chunk indices) are staged once in shared memory; the candidate list streams
// through a 256-entry shared ring refilled one 32-entry block ahead from a register-held load.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kRing = 256;

// The chain itself, run by ONE warp (shared by k_chain and k_small).  qoff / qcnt: queue layout of the chunk; s_q: the
// queues in shared memory; cand_o16: occupancy + table tag of every candidate GPU in canonical order (global memory,
// streamed through s_ring); log: one (key, candidate index) record per decision.  Returns the number of decisions.
template <int K>
__device__ __forceinline__ uint32_t chain_warp(const CandTab& tab, const uint32_t* qoff, const uint32_t* qcnt, const uint16_t* s_q, uint32_t* s_ring,
                                               const uint16_t* s_feas, const uint16_t* __restrict__ cand_o16, uint32_t n_cand, uint2* log,
                                               const uint32_t* __restrict__ heads_in, uint32_t* __restrict__ heads_out, uint32_t lane,
                                               uint32_t* visited_out, uint32_t* jumps_out) {
    uint32_t cmask[K], keylow[K], pbit[K], head[K], left[K], qa[K], tcur[K], tnext[K];
    bool reports[K];
    uint32_t rem = 0;                       // requests still pending over all profiles that have a candidate (warp-uniform)
    {
        uint32_t seen = 0;
        for (uint32_t k = 0; k < 4; ++k)
            for (uint32_t l = 0; l < 32; ++l) {
                const uint32_t d = tab.desc[k][l];
                if (!(d >> 31)) continue;
                const uint32_t p = d & 15u;
                if ((seen >> p) & 1u) continue;
                seen |= 1u << p;
                const uint32_t h = heads_in ? heads_in[p] : 0u, e = qcnt[p];
                rem += e > h ? e - h : 0u;
            }
    }
    const uint32_t rem0 = rem;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const uint32_t d = tab.desc[k][lane];
        const bool valid = d >> 31;
        const uint32_t p = d & 15u;
        cmask[k] = valid ? ((d >> 16) & 0xFFu) | (1u << (8 + ((d >> 24) & 7u))) : 0xFFFFu;      // slot mask + own-table bit
        keylow[k] = (p << 11) | (((d >> 4) & 7u) << 8) | (cmask[k] & 0xFFu);
        pbit[k] = valid ? 1u << p : 0u;
        reports[k] = valid && ((d >> 4) & 7u) == 0;       // first candidate of the row reports the head
        const uint32_t qb = qoff[p], end = valid ? qcnt[p] : 0u;
        head[k] = heads_in ? heads_in[p] : 0u;
        left[k] = end > head[k] ? end - head[k] : 0u;      // requests of this profile not yet popped
        qa[k] = qb + head[k];                              // shared-memory index of the current head entry
        tcur[k] = left[k] > 0 ? ((uint32_t)s_q[qa[k]] << 15) | keylow[k] : kInf;
        tnext[k] = left[k] > 1 ? ((uint32_t)s_q[qa[k] + 1] << 15) | keylow[k] : kInf;
    }
    auto ldc = [&](uint32_t idx) -> uint32_t { return idx < n_cand ? (uint32_t)__ldcg(cand_o16 + idx) : 0xFFFFu; };   // past the end: nothing fits
    uint32_t fill = 0, pending;
    auto reload = [&](uint32_t at) {       // synchronous (re)fill of 5 blocks starting at the block that holds `at`
        __syncwarp();                          // every lane is done reading the slots that are about to be overwritten
        fill = at & ~31u;
        for (int b = 0; b < 5; ++b) { s_ring[(fill + lane) & (kRing - 1)] = ldc(fill + lane); fill += 32; }
        pending = ldc(fill + lane);
        __syncwarp();
    };
    reload(0);
    uint32_t i0 = 0;
    uint32_t o0 = s_ring[0], o1 = s_ring[1], o2 = s_ring[2];
    uint32_t jumps = 0;
    uint2* lp = log;
    while (rem) {
        uint32_t key = kInf;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const uint32_t kk = (o0 & cmask[k]) == 0 ? tcur[k] : ((o1 & cmask[k]) == 0 ? tcur[k] | 0x80000000u : kInf);
            key = min(key, kk);
        }
        const uint32_t m = __reduce_min_sync(0xFFFFFFFFu, key);
        if (m == kInf) {
            // Neither GPU takes anything.  Ballot over the next candidates for one on which a profile that still has
            // pending requests fits (the list was built for every profile pending at chunk start).
            uint32_t alive = 0;
#pragma unroll
            for (int k = 0; k < K; ++k) alive |= tcur[k] != kInf ? pbit[k] : 0u;
            alive = __reduce_or_sync(0xFFFFFFFFu, alive);
            uint32_t j = i0 + 2;
            bool found = false;
            while (j < n_cand) {
                const uint32_t c = ldc(j + lane);                 // table = the one cleared bit of the tag
                const uint32_t b = __ballot_sync(0xFFFFFFFFu, c != 0xFFFFu && (s_feas[(__ffs(~(c >> 8) & 0xFFu) - 1) * 256 + (c & 0xFFu)] & alive) != 0);
                if (b) { j += __ffs(b) - 1; found = true; break; }
                j += 32;
            }
            ++jumps;
            if (!found) break;
            i0 = j;
            if (i0 + 64 > fill) reload(i0);
            o0 = s_ring[i0 & (kRing - 1)]; o1 = s_ring[(i0 + 1) & (kRing - 1)]; o2 = s_ring[(i0 + 2) & (kRing - 1)];
            continue;
        }
        const uint32_t sel = m >> 31;
        if (lane == 0) *lp = make_uint2(m, i0 + sel);     // decision log: (key, candidate index it landed on)
        ++lp;
        if (sel) {      // warp-uniform: the current GPU is finished, the next one becomes current
            o0 = o1 | (m & 0xFFu); o1 = o2;
            ++i0;
            o2 = s_ring[(i0 + 2) & (kRing - 1)];
            if ((i0 & 31u) == 0 && fill < i0 + 224) {
                __syncwarp();
                s_ring[(fill + lane) & (kRing - 1)] = pending;
                fill += 32;
                pending = ldc(fill + lane);
                __syncwarp();
            }
        } else {
            o0 |= m & 0xFFu;
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {       // lanes of the winning profile (same t, same profile field) pop their queue
            // branch-free: the shared-memory read is unconditional (index 0 when there is nothing to read)
            const bool adv = ((m ^ tcur[k]) & 0x7FFFF800u) == 0 && tcur[k] != kInf;
            left[k] -= adv ? 1u : 0u;
            qa[k] += adv ? 1u : 0u;
            const bool more = left[k] > 1;
            const uint32_t v = s_q[more ? qa[k] + 1 : 0u];
            const uint32_t tn = more ? (v << 15) | keylow[k] : kInf;
            tcur[k] = adv ? tnext[k] : tcur[k];
            tnext[k] = adv ? tn : tnext[k];
        }
        --rem;
    }
#pragma unroll
    for (int k = 0; k < K; ++k)
        if (reports[k] && heads_out) heads_out[(keylow[k] >> 11) & 15u] = qcnt[(keylow[k] >> 11) & 15u] - left[k];
    *visited_out = i0; *jumps_out = jumps;
    return rem0 - rem;
}

template <int K>
__global__ void __launch_bounds__(kChainThreads, 1) k_chain(CandTab tab, Ctrl* ctrl, const uint16_t* __restrict__ q_global,
                                                             const uint16_t* __restrict__ cand_o16, const uint16_t* __restrict__ feas,
                                                             uint2* __restrict__ log, const uint32_t* __restrict__ heads_in,
                                                             uint32_t* __restrict__ heads_out) {
    extern __shared__ __align__(16) uint16_t s_q[];
    __shared__ uint32_t s_ring[kRing];
    __shared__ uint16_t s_feas[kMaxTables * 256];
    if (__popc(ctrl->active) == 1) {        // single-profile chunk: the sweep kernels committed it in scan mode, nothing to chain
        if (threadIdx.x == 0) ctrl->n_log = 0;
        return;
    }
    const uint32_t q_total = ctrl->qoff[ISL_MAX_PROFILES];
    {   // stage every queue of the chunk: <= 129 KB, 16-byte vector copies
        const uint4* src = reinterpret_cast<const uint4*>(q_global);
        uint4* dst = reinterpret_cast<uint4*>(s_q);
        for (uint32_t i = threadIdx.x; i < (q_total + 7) / 8; i += kChainThreads) dst[i] = src[i];
        for (uint32_t i = threadIdx.x; i < kMaxTables * 256; i += kChainThreads) s_feas[i] = feas[i];
    }
    __syncthreads();
    if (!is_chain_warp(threadIdx.x >> 5)) return;
    uint32_t visited, jumps;
    const uint32_t steps = chain_warp<K>(tab, ctrl->qoff, ctrl->qcnt, s_q, s_ring, s_feas, cand_o16, ctrl->n_cand, log, heads_in, heads_out, threadIdx.x,
                                         &visited, &jumps);
    if (threadIdx.x == 0) {
        ctrl->n_log = steps;
        atomicAdd(&ctrl->placed, (unsigned long long)steps);
        atomicAdd(&ctrl->steps, (unsigned long long)steps);
        atomicAdd(&ctrl->visited, (unsigned long long)visited);
        atomicAdd(&ctrl->jumps, (unsigned long long)jumps);
    }
}

// ---------------------------------------------------------------------------------------------
// k_small<K>: the whole hot path of ONE small batch (<= 1024 requests) in ONE launch of ONE CTA — the latency path
// (BASELINE config 5: a reconciler handing over one or two pods at a time).  Same steps as the big path:
//   A  frees / default results / stable partition of the ALLOC requests into per-profile queues (shared memory)
//   B  vectorised sweep of the inventory with ordered compaction of the candidate GPUs (16 GPUs per thread and round)
//   C  the decision chain (warp 0)
//   D  commit of the logged decisions
// Tiny batches (<= 64 requests) arrive as kernel parameters and their results go straight to mapped pinned host memory,
// so the call is one launch and one stream synchronisation.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kSmallThreads = 1024;
constexpr uint32_t kSmallMax = 1024;              // requests: one per thread in phase A
constexpr uint32_t kSmallInline = 64;             // requests that travel as kernel parameters
struct SmallReqs { uint2 r[kSmallInline]; };

template <int K>
__global__ void __launch_bounds__(kSmallThreads, 1) k_small(CandTab tab, DevProfiles prof, uint32_t n, const uint2* __restrict__ in, SmallReqs inl,
                                                             uint2* __restrict__ out, uint8_t* __restrict__ occ, const uint8_t* __restrict__ gtab,
                                                             const uint16_t* __restrict__ feas, uint32_t G, uint32_t lo, uint32_t hi,
                                                             uint32_t cand_profiles, uint32_t* __restrict__ cand, uint16_t* __restrict__ cand_o16, Ctrl* stats) {
    __shared__ uint16_t s_q[kSmallMax + kQPad * ISL_MAX_PROFILES];
    __shared__ uint32_t s_ring[kRing];
    __shared__ uint16_t s_feas[kMaxTables * 256];
    __shared__ uint32_t s_seg[32][ISL_MAX_PROFILES];
    __shared__ uint32_t s_qoff[ISL_MAX_PROFILES + 1], s_qcnt[ISL_MAX_PROFILES], s_scan[32], s_active, s_base, s_nlog, s_freed;
    __shared__ uint2 s_log[kSmallMax];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t* occ32 = reinterpret_cast<uint32_t*>(occ);
    for (uint32_t i = tid; i < kMaxTables * 256; i += kSmallThreads) s_feas[i] = feas[i];
    if (tid < 32 * ISL_MAX_PROFILES) (&s_seg[0][0])[tid] = 0;
    if (tid == 0) { s_base = 0; s_freed = 0; }
    __syncthreads();
    // ---- A: one request per thread
    uint32_t key = kSkip, rank = 0;
    if (tid < n) {
        uint32_t gi, span;
        key = prepare_request(in ? in[tid] : inl.r[tid], out[tid], prof, G, lo, hi, gi, span);
        if (span) { atomicAnd(&occ32[gi >> 2], ~span); atomicAdd(&s_freed, 1u); }
    }
    {
        const uint32_t peers = __match_any_sync(0xFFFFFFFFu, key);
        rank = __popc(peers & ((1u << lane) - 1u));
        if (key != kSkip && lane == (uint32_t)(__ffs(peers) - 1)) s_seg[warp][key] = __popc(peers);
    }
    __syncthreads();
    if (tid < ISL_MAX_PROFILES) {           // exclusive scan over the 32 warps, in request order
        uint32_t run = 0;
        for (uint32_t w = 0; w < 32; ++w) { const uint32_t c = s_seg[w][tid]; s_seg[w][tid] = run; run += c; }
        s_qcnt[tid] = run;
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t off = 0, active = 0, allocs = 0;
        for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) {
            s_qoff[p] = off;
            if (s_qcnt[p] && ((cand_profiles >> p) & 1u)) active |= 1u << p;
            allocs += s_qcnt[p];
            off += (s_qcnt[p] + kQPad - 1) & ~(kQPad - 1);
        }
        s_qoff[ISL_MAX_PROFILES] = off; s_active = active;
        if (allocs) atomicAdd(&stats->allocs, (unsigned long long)allocs);
        if (s_freed) atomicAdd(&stats->freed, (unsigned long long)s_freed);
    }
    __threadfence();                        // the frees must be visible to the sweep's loads
    __syncthreads();
    if (key != kSkip) s_q[s_qoff[key] + s_seg[warp][key] + rank] = (uint16_t)tid;
    // ---- B: sweep, 16 GPUs per thread and round, ordered compaction into cand / cand_o16
    const uint32_t active = s_active;
    if (active) {
        for (uint32_t base = lo / (kSmallThreads * 16u) * (kSmallThreads * 16u); base < hi; base += kSmallThreads * 16u) {
            const uint32_t g0 = base + tid * 16u;
            uint4 v = make_uint4(0, 0, 0, 0), tv = make_uint4(0, 0, 0, 0);
            uint32_t mask = 0;
            if (g0 < hi && g0 + 16u > lo) {
                v = __ldcg(reinterpret_cast<const uint4*>(occ) + (g0 >> 4)); tv = __ldcg(reinterpret_cast<const uint4*>(gtab) + (g0 >> 4));
                mask = sweep_mask16(v, tv, s_feas, active, g0, lo, hi);
            }
            const uint32_t c = __popc(mask);
            uint32_t incl = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += t; }
            if (lane == 31) s_scan[warp] = incl;
            __syncthreads();
            if (warp == 0) {                    // exclusive scan of the 32 warp totals
                const uint32_t t = s_scan[lane];
                uint32_t x = t;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, d); if ((int)lane >= d) x += y; }
                s_scan[lane] = x - t;
                if (lane == 31) s_nlog = x;     // round total (s_nlog is reused as scratch here)
            }
            __syncthreads();
            emit_candidates(mask, v, tv, g0, s_base + s_scan[warp] + incl - c, cand, cand_o16);
            __syncthreads();
            if (tid == 0) s_base += s_nlog;
            __syncthreads();
        }
    }
    __threadfence();
    __syncthreads();
    // ---- C: the chain
    if (is_chain_warp(warp)) {
        uint32_t visited = 0, jumps = 0;
        const uint32_t steps = active ? chain_warp<K>(tab, s_qoff, s_qcnt, s_q, s_ring, s_feas, cand_o16, s_base, s_log, nullptr, nullptr, lane, &visited, &jumps) : 0u;
        if (lane == 0) {
            s_nlog = steps;
            if (steps) { atomicAdd(&stats->placed, (unsigned long long)steps); atomicAdd(&stats->steps, (unsigned long long)steps); }
            if (visited) atomicAdd(&stats->visited, (unsigned long long)visited);
            if (jumps) atomicAdd(&stats->jumps, (unsigned long long)jumps);
        }
    }
    __syncthreads();
    // ---- D: commit
    for (uint32_t j = tid; j < s_nlog; j += kSmallThreads) commit_decision(s_log[j], cand, occ32, out, prof.flip);
}

// ---------------------------------------------------------------------------------------------
// k_few: the latency path of a reconciler that hands over one or two pods at a time (BASELINE configs 1 and 5): at most
// kFewMax requests, an inventory range of at most kFewGpus GPUs, first-fit.  Request-major on purpose — with a handful of
// requests there is nothing to amortise a partition / sweep / chain over: ONE CTA holds 16 occupancy bytes per thread in
// registers, the first-start tables in shared memory, and for every ALLOC in order finds the first feasible GPU with a
// block-wide min (redux + one shared-memory hop) — exactly the reference's scan order (:240-262, :303-384).  Requests travel as
// kernel parameters, results go straight to mapped pinned host memory: one launch, one stream synchronisation.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kFewThreads = 1024;
constexpr uint32_t kFewMax = 8;
constexpr uint32_t kFewGpus = kFewThreads * 16;

__global__ void __launch_bounds__(kFewThreads, 1) k_few(DevProfiles prof, uint32_t n, SmallReqs inl, uint2* __restrict__ out, uint8_t* __restrict__ occ,
                                                         const uint8_t* __restrict__ gtab, const uint8_t* __restrict__ lut, const uint8_t* __restrict__ sizes,
                                                         uint32_t n_tables, uint32_t G, uint32_t lo, uint32_t hi, Ctrl* stats) {
    __shared__ __align__(16) uint8_t s_lut[kMaxTables * ISL_MAX_PROFILES * 256];
    __shared__ uint8_t s_sizes[kMaxTables * ISL_MAX_PROFILES];
    __shared__ uint32_t s_red[32], s_win;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t* occ32 = reinterpret_cast<uint32_t*>(occ);
    for (uint32_t i = tid; i < n_tables * ISL_MAX_PROFILES * 64; i += kFewThreads) reinterpret_cast<uint32_t*>(s_lut)[i] = reinterpret_cast<const uint32_t*>(lut)[i];
    if (tid < n_tables * ISL_MAX_PROFILES) s_sizes[tid] = sizes[tid];
    uint32_t freed = 0, allocs = 0;
    if (tid < n) {          // defaults and FREEs, one request per thread
        uint32_t gi, span;
        allocs = prepare_request(inl.r[tid], out[tid], prof, G, lo, hi, gi, span) != kSkip;
        if (span) { atomicAnd(&occ32[gi >> 2], ~span); freed = 1; }
    }
    __threadfence();                        // the frees must be visible to the loads below
    __syncthreads();
    // 16 GPUs per thread, aligned to 16: the byte of a GPU outside [lo, hi) reads as full
    const uint32_t g0 = (lo & ~15u) + tid * 16u;
    uint4 v = make_uint4(~0u, ~0u, ~0u, ~0u), tv = make_uint4(0, 0, 0, 0);
    if (g0 < hi) { v = __ldcg(reinterpret_cast<const uint4*>(occ) + (g0 >> 4)); if (n_tables > 1) tv = __ldcg(reinterpret_cast<const uint4*>(gtab) + (g0 >> 4)); }
    uint32_t wv[4] = {v.x, v.y, v.z, v.w};
    const uint32_t twv[4] = {tv.x, tv.y, tv.z, tv.w};
    for (uint32_t r = 0; r < n; ++r) {      // the ALLOCs strictly in request order, each seeing all earlier commits
        const uint32_t w = inl.r[r].y, p = w & 0xFFu, op = (w >> 8) & 0xFFu;
        if (op != ISL_OP_ALLOC || p >= prof.n) continue;        // uniform
        uint32_t best = kInf;
#pragma unroll
        for (int j = 15; j >= 0; --j) {     // descending, so the lowest feasible GPU of the thread is what remains
            const uint32_t g = g0 + j, o = byte16(wv, j), t = byte16(twv, j) & (kMaxTables - 1);
            if (g >= lo && g < hi && s_lut[(t * ISL_MAX_PROFILES + p) * 256 + o] != ISL_START_NONE) best = g;
        }
        const uint32_t wm = __reduce_min_sync(0xFFFFFFFFu, best);
        if (lane == 0) s_red[warp] = wm;
        __syncthreads();
        if (warp == 0) { const uint32_t m = __reduce_min_sync(0xFFFFFFFFu, s_red[lane]); if (lane == 0) s_win = m; }
        __syncthreads();
        const uint32_t g = s_win;
        if (g != kInf && g >= g0 && g < g0 + 16u) {             // the owner commits
            const uint32_t j = g - g0, sh = (j & 3u) * 8u, o = byte16(wv, j), t = byte16(twv, j) & (kMaxTables - 1);
            const uint32_t st = s_lut[(t * ISL_MAX_PROFILES + p) * 256 + o], size = s_sizes[t * ISL_MAX_PROFILES + p];
            const uint32_t o2 = o | slice_span(st, size);
            wv[j >> 2] = (wv[j >> 2] & ~(0xFFu << sh)) | (o2 << sh);
            occ[g] = (uint8_t)o2;
            out[r] = pack_result(flip_gpu(g, prof.flip), st, size, ISL_ST_PLACED);
            atomicAdd(&stats->placed, 1ull); atomicAdd(&stats->steps, 1ull);
        }
        // s_red / s_win are rewritten only after the next request's first barrier has been passed by everybody who read them
    }
    // statistics (off the caller's critical path: the results are already on their way)
    if (freed) atomicAdd(&stats->freed, 1ull);
    if (allocs) atomicAdd(&stats->allocs, 1ull);
}

// ---------------------------------------------------------------------------------------------
// k_commit: one thread per logged decision: the result record of its request (the fields of
// AllocationDetails the allocator decides) and the slot mask ORed into the packed occupancy word.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_commit(const Ctrl* __restrict__ ctrl, const uint2* __restrict__ log, const uint32_t* __restrict__ cand,
                                                 uint32_t* __restrict__ occ32, uint2* __restrict__ out_chunk, uint32_t flip) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < ctrl->n_log) commit_decision(log[j], cand, occ32, out_chunk, flip);
}

// ---------------------------------------------------------------------------------------------
// k_pipeline<K>: the segment pipeline for STREAMS of batches (BASELINE config 4's shape).
//
// The commit chain of one chunk is sequential, but chunks of a stream pipeline exactly over inventory segments: segment s may work on
// chunk c+1 while segment s+1 is still on chunk c, because inside a segment everything happens in stream order (occupancy of the
// segment lives in this CTA's shared memory), and the only state that crosses a segment boundary is the per-profile queue-head token.
// One persistent CTA per segment (cooperative launch, all co-resident; one CTA fills an SM's shared memory).  Per chunk a CTA
//   0. has the chunk's queues copied into shared memory by cp.async when the previous chunk's chain ended      queue_load_async
//   1. applies the batch's frees that fall into its range                                                       apply_frees
//   2. sweeps its occupancy bytes into an ordered candidate list, before the token arrives                     sweep_subsegment
//   3. takes its entry heads: the token of segment s-1 (self-validating words: epoch tag + head, polled by 16 lanes), or in the
//      speculative rounds a prediction; converts the queue windows it may pop into ready-made keys     read_entry, stage_windows
//   4. runs the decision chain on its candidates (warp 0; DESIGN.md 4.1) and                                     decide
//   5. publishes the token for segment s+1 (speculative rounds: exchanges records until certified)       exchange_round
//   6. commits the logged decisions: result records + occupancy bits                                            commit_log
// resolve_plain and resolve_rounds run steps 3-5.  Host-buffer streams: the batches are fed by a second stream while this kernel runs
// (wait_ready), an extra CTA delivers finished chunks into the caller's pinned result array (deliver_chunks).
// Results are bit-identical to resolving the batches one after the other.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kSegMax = 512;                   // GPUs per (sub-)segment (2 per thread in the local sweep)
constexpr uint32_t kSubMax = 8;                     // sub-segments one CTA walks per chunk: inventories beyond SMs x 512 GPUs stay on the pipeline
constexpr uint32_t kPipeThreads = 256;              // 1 or 2 GPUs per thread in the local sweep
static_assert(kPipeThreads == kSegMax || 2 * kPipeThreads == kSegMax, "sweep layout");
constexpr uint32_t kLogCap = 8 * kSegMax;           // a GPU accepts at most 8 placements
constexpr uint32_t kTokStride = 32;                 // uint32 per token: 16 tagged head words (token_tag inside a GPU, xtoken_tag across GPUs)
// shared memory: occupancy bytes | candidate records (+8 sentinels) | decision log (+1 pseudo-decision) | the chunk's queues (uint16) | queue-window keys
constexpr uint32_t kPipeOffCand = kSegMax * kSubMax;      // occupancy bytes of the whole stage (all its sub-segments)
constexpr uint32_t kCandPad = 16;                   // INF records behind a segment's candidates: a group of pseudo-decisions may walk that far
constexpr uint32_t kWinPad = 10;                    // INF keys behind every queue window: an exhausted lane is popped at most once per decision of a group
constexpr uint32_t kPipeOffLog = kPipeOffCand + 4 * (kSegMax + kCandPad);
constexpr uint32_t kPipeOffQ = (kPipeOffLog + 8 * (kLogCap + 1) + 15u) & ~15u;
constexpr uint32_t kPipeOffWin = kPipeOffQ + 2 * kQCap + 16;
constexpr uint32_t kWinTotal = 12288;               // 32-bit queue-window keys a segment can stage for all profiles together
constexpr uint32_t kPipeSmem = kPipeOffWin + 4 * (kWinTotal + 4 * ISL_MAX_PROFILES);

// largest segment whose worst-case queue windows (every candidate GPU accepting every legal start of every
// profile) fit: n_cand * total_candidates + 2 sentinels per profile <= kWinTotal
constexpr uint32_t kWinMargin = 32;                 // speculative rounds: queue entries staged on either side of a window, so that a corrected entry nearby re-uses it
__host__ __device__ inline uint32_t max_segment_for(uint32_t total_candidates) {
    const uint32_t s = (kWinTotal - (kWinPad + 2 * kWinMargin + 2) * ISL_MAX_PROFILES) / (total_candidates ? total_candidates : 1u);
    return s >= kSegMax ? kSegMax : s / 64u * 64u;
}

struct ChunkDesc {
    uint32_t req_off, n, batch, first_of_batch;
    uint2* host_out;                // open streams: mapped pinned destination of this chunk's results (nullptr: PipeArgs.host_out + req_off)
    uint64_t pad;
};

struct PipeArgs {
    uint32_t n_chunks, n_seg, seg, lo, hi, epoch;     // seg: GPUs per pipeline stage (CTA) = sub x sub-segments
    uint32_t sub;                                     // GPUs per sub-segment (<= kSegMax): what one sweep / chain / commit round covers
    const ChunkDesc* chunks;
    const Ctrl* cctl;               // per chunk: qoff / qcnt / active (written by k_partition)
    const uint16_t* q_all;          // per chunk queues, stride q_stride entries
    const uint8_t* free_acc;        // per batch one byte per GPU: OR of the slot masks its FREEs release (stride free_stride bytes)
    uint32_t q_stride, free_stride;
    uint32_t* tokens;               // [chunk][segment + 1][kTokStride] of (epoch tag << 17 | head); slot n_seg = 'everything placeable is placed' broadcast
    uint8_t* occ;
    const uint8_t* gtab;            // table id of every GPU's node
    uint2* out;
    const uint16_t* feas;
    Ctrl* stats;
    // partitioned inventory: the token crosses GPUs through peer-mapped memory (NVLink), one relaxed system-scope store per head word
    const uint32_t* inbox;          // local [chunk][kTokStride] of tagged head words, written by the previous rank's last segment (nullptr = first rank); cleared by the reader
    uint32_t* outbox;               // the next rank's inbox, peer-mapped (nullptr = last rank)
    uint32_t xepoch;                // stream id shared by all ranks
    // host-buffer streams (isl_place_stream): the batches are fed while the pipeline runs, the results leave chunk by chunk
    const uint32_t* ready;          // [batch] == epoch once the batch's requests are in HBM and its pre-pass is done (nullptr = all ready)
    uint32_t* done_cnt;             // [chunk] segments that have committed the chunk (zeroed per call; nullptr = no copier CTA)
    uint2* host_out;                // mapped pinned result array of the caller: CTA n_seg copies every complete chunk there
    // open streams (isl_stream_open / _submit / _wait / _close): batches arrive while the kernel runs, one chunk per batch, n_chunks is
    // the capacity; ready[b] == ~epoch closes the stream.  host_done[c] = epoch (mapped pinned) tells the host that chunk c is delivered.
    uint32_t open, copier;          // copier: an extra CTA (index n_seg) delivers finished chunks to host memory
    uint32_t* host_done;
    // causal window: chunk c may start only after chunk c - window has been committed by every segment (0 = no constraint)
    uint32_t window;
    unsigned long long wait_ns;     // a starved wait traps after this long instead of hanging the GPU
    // partitioned inventory, results gathered on the owner rank: peer-mapped result array of rank 0 (nullptr = keep results local)
    uint2* owner_out;
    // causal window across ranks: the CTA that completes a chunk on its rank adds 1 to ring_done[chunk] on the owner rank (peer atomic);
    // the owner starts chunk c only when ring_done[c - window] == world
    uint32_t* ring_done; uint32_t world;
    uint32_t flip;                  // ISL_POLICY_RIGHT_TO_LEFT: G, the reported GPU is G - 1 - internal index
    unsigned long long* trace;      // optional [chunk][segment][kTraceWords]: globaltimer ns of sweep done, token in, token out, commit done, chain start, chain end; decisions; jumps | visited << 32; ns of heads done, windows staged; 2 spare
    // speculative rounds (below): every stage simulates its segment from PREDICTED queue heads at once, the predictions are corrected round
    // by round and a stage commits once its entry heads are certified to be the true ones.  Record memory: spec_mem(), kSpecWordsPerChunk per chunk.
    uint32_t spec;
    unsigned long long* spec_mem;
    // partitioned inventory: the stages of all ranks form ONE sequence (global index spec_base + stage); every rank keeps the whole record
    // memory and a stage stores what later ranks read straight into their copies (peer stores over NVLink, system scope)
    uint32_t spec_world, spec_rank, spec_base, spec_total;
    unsigned long long* spec_peer[8];
    unsigned long long* spec_dbg;   // optional [kSpecRounds][8] globaltimer stamps of the rounds of ONE (chunk, stage) cell (ISL_SPEC_DBG=chunk,stage; tools/spec_trace.py)
    uint32_t spec_dbg_cell;         // chunk << 16 | stage
};

// ---------------------------------------------------------------------------------------------
// Speculative rounds over the stages of ONE chunk (DESIGN.md 4.5) — exact, only faster.
// A chunk's decisions are one recurrence over the inventory: stage s needs the queue heads stage s-1 leaves (the token).  Instead of
// idling until the token has travelled, every stage simulates its segment at once from a PREDICTED token:
//   round 0   every stage publishes what its occupancy can take (per contention group: placements of the size >= 4 profiles, slices left
//             for the size 1/2 profiles); stage s predicts its entry heads from the sums over the stages in front of it
//   round r   stage s simulates from its predicted entry H (the exact chain of 4.1, log kept in shared memory), publishes its exit heads
//             X (to s+1) and the group masses it consumed D (to every later stage), reads X of s-1 and D of all j < s, and corrects:
//             H' = X(s-1) shifted, per group, to the mass sum of D(j), j < s   (a Newton step: a shift of the entry by conserved
//             quantities passes through a segment unchanged; the split inside a group heals by itself within a few hundred GPUs)
//   stage s is CERTIFIED in round r when H(j) of round r-1 equalled X(j-1) of round r-1 for every j <= s: by induction from stage 0
//             (whose entry is the true one) every such entry is the true token; it commits its log and publishes final records.
// Every round certifies at least one more stage, so the worst case is the token travelling stage by stage as before; predictions that
// hold certify whole runs of stages at once.  Words are self-validating (call epoch and round above the payload): no flags, no fences.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kSpecMaxStages = 148;            // stages of one speculative sequence (over all ranks of a partitioned inventory)
constexpr uint32_t kSpecStride = 160;               // stage slots per row (>= kSpecMaxStages)
constexpr uint32_t kSpecRounds = 160;               // rounds <= stages + 2
constexpr uint32_t kSpecWordsPerChunk = kSpecStride * (32 + 16 + kSpecRounds + 1 + 2 + 1);
struct SpecMem {
    unsigned long long* x;          // [stage][round & 1][16]   tag(round) << 32 | exit head
    unsigned long long* xf;         // [stage][16]              final: tagF << 32 | certified-in-round << 24 | exit head
    unsigned long long* d;          // [round][stage]           tag(round) << 32 | c << 31 | dq << 13 | dr   (c: entry equalled the predecessor's exit one round earlier)
    unsigned long long* df;         // [stage]                  final: tagF << 32 | certified-in-round << 24 | dq << 13 | dr
    unsigned long long* m;          // [stage][2]               round 0: tag(0) << 32 | placements of the big group ; tag(0) << 32 | slices with << 16 | slices without them
    unsigned long long* ack;        // [stage]                  epoch << 32 | last round whose X(stage - 1) this stage has read
};
__host__ __device__ inline SpecMem spec_mem(unsigned long long* base, uint32_t chunk) {
    unsigned long long* p = base + (size_t)chunk * kSpecWordsPerChunk;
    SpecMem s;
    s.x = p; p += kSpecStride * 32; s.xf = p; p += kSpecStride * 16; s.d = p; p += (size_t)kSpecStride * kSpecRounds;
    s.df = p; p += kSpecStride; s.m = p; p += kSpecStride * 2; s.ack = p;
    return s;
}

constexpr uint32_t kTraceWords = 12;
constexpr int kUnroll = 8;                   // decisions per trip of the decision loop
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// Trace stamp without a branch: a divergent `if (lane == 0)` in front of the decision loop can leave warp 0 split for good, and
// every redux of the loop then takes the BRA.DIV emulation path (several times slower decisions).  `p` may be any address when !pred.
__device__ __forceinline__ void stamp_if(bool pred, unsigned long long* p) {
    asm volatile("{ .reg .pred q; .reg .u64 t; setp.ne.u32 q, %0, 0; mov.u64 t, %%globaltimer; @q st.global.u64 [%1], t; }" ::"r"((uint32_t)pred), "l"(p) : "memory");
}
__device__ __forceinline__ void store_if(bool pred, unsigned long long* p, unsigned long long v) {
    asm volatile("{ .reg .pred q; setp.ne.u32 q, %0, 0; @q st.global.u64 [%1], %2; }" ::"r"((uint32_t)pred), "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_gpu(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_gpu(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ld_relaxed_gpu_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_relaxed_sys_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Speculative rounds: move the heads of the profiles in `members` so that their mass (sum of weight x head) changes by d.
// By a whole warp: lane p < 16 holds head h of profile p and returns the moved head.  Shares proportional to the queue lengths; the single-slice profile with the highest index (a group without one:
// its highest member) takes the remainder, so that the mass is met exactly whenever the weights allow it.  |d| <= 2^13: float shares.
__device__ __forceinline__ uint32_t spec_spread_warp(uint32_t h, uint32_t qc, uint32_t w, uint32_t members, int d, bool weighted, uint32_t lane) {
    const bool in = (members >> lane) & 1u;
    if (!weighted) w = 1;
    const uint32_t light = __ballot_sync(0xFFFFFFFFu, in && w <= 1), heavy = __ballot_sync(0xFFFFFFFFu, in && w > 1);
    const uint32_t tot = __reduce_add_sync(0xFFFFFFFFu, in ? qc * w : 0u);
    if (d == 0 || members == 0) return h;
    const uint32_t last = 31u - __clz(light ? light : heavy);
    int dp = in && lane != last && tot ? __float2int_rn((float)d * (float)qc / (float)tot) : 0;
    const int used = __reduce_add_sync(0xFFFFFFFFu, dp * (int)w);
    const int wl = (int)__shfl_sync(0xFFFFFFFFu, w, last);
    if (lane == last) dp = (d - used) / wl;
    if (!in) return h;
    const int v = (int)h + dp;
    return (uint32_t)(v < 0 ? 0 : (v > (int)qc ? (int)qc : v));
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t sa) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(sa)); return v; }
__device__ __forceinline__ uint32_t lds_u16(uint32_t sa) { uint32_t v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(sa)); return v; }
__device__ __forceinline__ void sts_v2_if(bool pred, uint32_t sa, uint32_t x, uint32_t y) {
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %0, 0; @p st.shared.v2.u32 [%1], {%2, %3}; }" ::"r"((uint32_t)pred), "r"(sa), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ uint32_t add_if(bool pred, uint32_t x, uint32_t inc) {         // one predicated add instead of select + move
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %1, 0; @p add.u32 %0, %0, %2; }" : "+r"(x) : "r"((uint32_t)pred), "r"(inc));
    return x;
}
__device__ __forceinline__ uint32_t redux_min_u32(uint32_t v) {
    uint32_t r;
    asm volatile("redux.sync.min.u32 %0, %1, 0xffffffff;" : "=r"(r) : "r"(v));
    return r;
}
__device__ __forceinline__ uint32_t lds_u32_if(bool pred, uint32_t sa, uint32_t keep) {   // predicated load: keeps `keep` when !pred
    asm volatile("{ .reg .pred p; setp.ne.u32 p, %1, 0; @p ld.shared.u32 %0, [%2]; }" : "+r"(keep) : "r"((uint32_t)pred), "r"(sa));
    return keep;
}

// Rare path of the decision chain, kept out of line so that the hot loop stays free of divergence-capable constructs:
// first candidate index >= from + 2 on which a profile of `alive` fits, or kInf.
__device__ __noinline__ uint32_t pipeline_skip(uint32_t sa_cand, const uint16_t* s_feas, uint32_t n_cand, uint32_t cur_plus2, uint32_t alive, uint32_t lane) {
    alive = __reduce_or_sync(0xFFFFFFFFu, alive);
    uint32_t j = cur_plus2;                      // record index of (current + 2)
    while (alive && j < n_cand) {
        const uint32_t cr = j + lane < n_cand ? lds_u32(sa_cand + 4 * (j + lane)) : kInf;
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, cr != kInf && (s_feas[(__ffs(~(cr >> 8) & 0xFFu) - 1) * 256 + (cr & 0xFFu)] & alive) != 0);
        if (b) return j + __ffs(b) - 1;
        j += 32;
    }
    return kInf;
}

// A head word of a token is self-validating: a 15-bit tag above its 17 bits of payload (heads <= 65 536).  Inside a GPU the tag is the
// call's epoch; across GPUs it is the stream id all ranks share, never 0, so that a cleared inbox slot is never valid.
__device__ __forceinline__ uint32_t token_tag(const PipeArgs& a) { return a.epoch & 0x7FFFu; }
__device__ __forceinline__ uint32_t xtoken_tag(const PipeArgs& a) { return a.xepoch % 32767u + 1u; }
__device__ __forceinline__ uint32_t tag_word(uint32_t tag, uint32_t h) { return (tag << 17) | h; }

// Lane p < 16: head h of profile p leaves stage seg for chunk c — the word the next stage polls and, behind the last stage, the word in
// the next rank's inbox
__device__ __forceinline__ void publish_token(const PipeArgs& a, uint32_t c, uint32_t seg, uint32_t lane, uint32_t h) {
    uint32_t* tok = a.tokens + ((size_t)c * (a.n_seg + 1) + seg) * kTokStride;
    uint32_t* peer = seg == a.n_seg - 1 && a.outbox ? a.outbox + (size_t)c * kTokStride : nullptr;
    st_relaxed_gpu(tok + lane, tag_word(token_tag(a), h));
    if (peer) st_relaxed_sys(peer + lane, tag_word(xtoken_tag(a), h));
}

// The one bounded wait of the pipeline: polls until poll() holds, sleeping sleep_ns between polls (0: spin).  A wait that starves for
// deadline_ns (from t0) traps instead of hanging the GPU; the clock is read every 256th poll only.  A __trap ends the whole grid, so every
// chain of stages that wait on each other ends in such a wait: the in-GPU token poll (read_entry) has no deadline of its own.
template <typename Poll>
__device__ __forceinline__ void wait_until(Poll poll, unsigned long long deadline_ns, uint32_t sleep_ns, unsigned long long t0 = globaltimer_ns()) {
    for (uint32_t n = 1; !poll(); ++n) {
        if (sleep_ns) __nanosleep(sleep_ns);
        if ((n & 255u) == 0 && globaltimer_ns() - t0 > deadline_ns) __trap();
    }
}

// A stage's shared state beside the dynamic buffers (kPipeSmem).  The plain instantiations never touch SpecShared: it takes no shared
// memory there.
struct PipeShared {
    uint16_t feas[kMaxTables * 256];
    uint8_t tab[kSegMax * kSubMax];                 // table of every local GPU
    uint32_t heads[ISL_MAX_PROFILES], wn[ISL_MAX_PROFILES], wbase[ISL_MAX_PROFILES], qbeg[ISL_MAX_PROFILES], pop[ISL_MAX_PROFILES];
    uint32_t maxacc[ISL_MAX_PROFILES], minsize[ISL_MAX_PROFILES], usable[kMaxTables], plist[ISL_MAX_PROFILES], nplist;
    uint32_t warp[kPipeThreads / 32], ncand, nfree, nlog, idle, closed, cap;
};
struct SpecShared {
    // predicted entry heads, own / predecessor's exit heads, queue lengths and offsets, gathered sums, contention groups
    uint32_t specH[ISL_MAX_PROFILES], specX[ISL_MAX_PROFILES], specXp[ISL_MAX_PROFILES], qc[ISL_MAX_PROFILES], qo[ISL_MAX_PROFILES];
    uint32_t acc[4], grp_big, grp_small, specflag, bigd[32], nbigd, dqr[2], us[kMaxTables];
    uint8_t smallm[kMaxTables][ISL_MAX_PROFILES];
    // staged key windows outlive a simulation: per profile the first staged queue position, the staged entries, the entry's place among them
    uint32_t wlo[ISL_MAX_PROFILES], wlen[ISL_MAX_PROFILES], woff[ISL_MAX_PROFILES], wvalid, restage;
    // the c bit of the stage right in front; both correction rules' candidates of the previous round (Newton step, plain chaining)
    uint32_t predc, predA[ISL_MAX_PROFILES], predB[ISL_MAX_PROFILES], havepred;
    // bounded simulations: entry / exit heads of the last COMPLETE simulation; {decisions of the largest complete one, have one, the log
    // in shared memory is a complete simulation of the current entry}; this simulation was cut off
    uint32_t Hc[ISL_MAX_PROFILES], Xc[ISL_MAX_PROFILES], capst[3], capped;
};

struct Stage {                      // a pipeline stage (CTA): its GPUs and its dynamic shared buffers (kPipeSmem), with their shared addresses
    uint32_t seg, lo, n_g, sa_cand, sa_log, sa_q, sa_wkey;
    uint32_t *occ32, *cand, *wkey;  // occupancy bytes of all sub-segments; records (local gpu << 16 | table tag | occ) + sentinels; key windows
    uint2* log;                     // (key, candidate index) per decision
    const uint16_t* q;              // the chunk's queues: uint16 in-chunk request indices
};
struct PipeCounters { unsigned long long steps, jumps, visited, sims, rounds_sum, cells, spec_steps, spec_visited; };
template <int K>
struct ChainSlots {                 // chain-warp constants: one (profile, start) candidate per slot
    uint32_t cmask[K], klow[K], cprof[K];
    bool valid[K], reports[K];
    __device__ __forceinline__ ChainSlots(const CandTab& tab, uint32_t lane) {
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const uint32_t d = tab.desc[k][lane];
            valid[k] = d >> 31;
            cprof[k] = d & 15u;
            cmask[k] = valid[k] ? ((d >> 16) & 0xFFu) | (1u << (8 + ((d >> 24) & 7u))) : 0xFFFFu;   // slot mask + own-table bit
            klow[k] = (((d >> 4) & 7u) << 8) | (cmask[k] & 0xFFu);            // order-in-row and slot mask; t and profile come from the window key
            reports[k] = valid[k] && ((d >> 4) & 7u) == 0;
        }
    }
};
struct Rounds {                     // one speculative cell's way through the rounds
    SpecMem sm;
    unsigned long long tagb, tagF, p_word, t_cell, sims_cell;     // spec trace: [0] sweep + prediction done, [7] simulations
    uint32_t tage, gseg, gtot, rnd;                               // gseg: my place in the sequence of all stages of all ranks
    bool c_prev, need_sim, known_exact, p_final;                  // p_final: the pollers' certified stage's final record is kept in p_word
};

// Record words of the rounds: a partitioned inventory reads and writes them at system scope
__device__ __forceinline__ unsigned long long spec_ld(const PipeArgs& a, const unsigned long long* p) { return a.spec_world > 1 ? ld_relaxed_sys_u64(p) : ld_relaxed_gpu_u64(p); }
// a word every LATER stage reads: my copy and the copies of the ranks behind me
__device__ __forceinline__ void spec_pub_down(const PipeArgs& a, unsigned long long* p, unsigned long long v) {
    st_relaxed_gpu_u64(p, v);
    if (a.spec_world > 1) for (uint32_t r = a.spec_rank + 1; r < a.spec_world; ++r) st_relaxed_sys_u64(a.spec_peer[r] + (p - a.spec_mem), v);
}
// a word only the next (prev = false) / the previous (prev = true) stage reads
__device__ __forceinline__ void spec_pub_nb(const PipeArgs& a, uint32_t seg, unsigned long long* p, unsigned long long v, bool prev) {
    const bool remote = a.spec_world > 1 && (prev ? (seg == 0 && a.spec_rank > 0) : (seg + 1 == a.n_seg && a.spec_rank + 1 < a.spec_world));
    if (remote) st_relaxed_sys_u64(a.spec_peer[prev ? a.spec_rank - 1 : a.spec_rank + 1] + (p - a.spec_mem), v);
    else st_relaxed_gpu_u64(p, v);
}
// Round rnd's record at p, or — once its stage is certified — that stage's final record at pf, which stands for every round from then on
// and is read once
__device__ __forceinline__ unsigned long long read_record(const PipeArgs& a, const unsigned long long* p, const unsigned long long* pf,
                                                          unsigned long long tagr, Rounds& r) {
    if (r.p_final) return r.p_word;
    unsigned long long w;
    uint32_t polls = 0;
    wait_until([&] {
        w = spec_ld(a, p);
        if ((w >> 32) == (tagr >> 32)) return true;
        if ((polls++ & 3u) != 0) return false;
        w = spec_ld(a, pf);
        r.p_final = (w >> 32) == (r.tagF >> 32) && ((w >> 24) & 0xFFu) <= r.rnd;
        return r.p_final;
    }, a.wait_ns, 0);
    if (r.p_final) r.p_word = w;
    return w;
}
// The X slot of round rnd - 2 is about to be overwritten: the successor must have read it (it has, as a rule)
__device__ __forceinline__ void wait_ack(const PipeArgs& a, const Rounds& r) {
    wait_until([&] { const unsigned long long w = spec_ld(a, r.sm.ack + r.gseg + 1); return (uint32_t)(w >> 32) == r.tage && (uint32_t)w + 2u >= r.rnd; }, a.wait_ns, 0);
}
// By warp 0, lane p < 16 for profile p: the masses of per-profile counts v (placements of the big group, slices of the small group),
// and the heads h moved so that the masses change by dq / dr (spec_spread_warp)
__device__ __forceinline__ void group_masses(uint32_t v, const PipeShared& s, const SpecShared& ss, uint32_t lane, uint32_t& q, uint32_t& r) {
    q = __reduce_add_sync(0xFFFFFFFFu, lane < ISL_MAX_PROFILES && ((ss.grp_big >> lane) & 1u) ? v : 0u);
    r = __reduce_add_sync(0xFFFFFFFFu, lane < ISL_MAX_PROFILES && ((ss.grp_small >> lane) & 1u) ? v * s.minsize[lane] : 0u);
}
__device__ __forceinline__ uint32_t shift_groups(uint32_t h, const PipeShared& s, const SpecShared& ss, int dq, int dr, uint32_t lane) {
    const uint32_t qc = lane < ISL_MAX_PROFILES ? ss.qc[lane] : 0u, w = lane < ISL_MAX_PROFILES ? s.minsize[lane] : 1u;
    h = spec_spread_warp(h, qc, w, ss.grp_big, dq, false, lane);
    return spec_spread_warp(h, qc, w, ss.grp_small, dr, true, lane);
}

// The extra CTA of a host-buffer stream (index n_seg): every chunk all segments have committed goes to the caller's (mapped, pinned)
// result array right away, so the D2H of the results hides behind the rest of the stream
__device__ __forceinline__ void deliver_chunks(const PipeArgs& a) {
    __shared__ uint32_t s_stop;
    const uint32_t tid = threadIdx.x;
    for (uint32_t c = 0; c < a.n_chunks; ++c) {
        if (tid == 0) {
            uint32_t stop = 0;
            wait_until([&] {        // 5 s beyond the stages' deadline: a starved stage traps first
                if (ld_acquire_gpu(a.done_cnt + c) >= a.n_seg) return true;
                // a closed (or aborted) stream never commits this chunk: ready[batch] holds ~epoch
                stop = a.ready && ld_acquire_gpu(a.ready + (a.open ? c : a.chunks[c].batch)) == ~a.epoch;
                return stop != 0;
            }, a.wait_ns + 5000000000ull, 256);
            s_stop = stop;
        }
        __syncthreads();
        if (s_stop) break;
        const ChunkDesc cd = a.chunks[c];
        const uint2* __restrict__ src = a.out + cd.req_off;
        uint2* __restrict__ dst = cd.host_out ? cd.host_out : a.host_out + cd.req_off;
        // 16-byte body between an 8-byte head / tail when source and destination are 16-byte aligned at the same records;
        // otherwise (a destination that is only 8-byte aligned relative to the staging buffer) plain 8-byte stores
        const bool same = ((reinterpret_cast<uintptr_t>(src) ^ reinterpret_cast<uintptr_t>(dst)) & 8u) == 0;
        if (same) {
            const uint32_t head = min(cd.n, (uint32_t)((reinterpret_cast<uintptr_t>(dst) >> 3) & 1u)), pairs = (cd.n - head) >> 1;
            if (tid == 0 && head) dst[0] = __ldcg(src);
            const uint4* __restrict__ s4 = reinterpret_cast<const uint4*>(src + head);
            uint4* __restrict__ d4 = reinterpret_cast<uint4*>(dst + head);
#pragma unroll 4
            for (uint32_t i = tid; i < pairs; i += kPipeThreads) d4[i] = __ldcg(s4 + i);
            if (tid == 0 && ((cd.n - head) & 1u)) dst[cd.n - 1] = __ldcg(src + cd.n - 1);
        } else {
#pragma unroll 4
            for (uint32_t i = tid; i < cd.n; i += kPipeThreads) dst[i] = __ldcg(src + i);
        }
        if (a.host_done) {          // the host may read the chunk's results as soon as it sees this word
            __threadfence_system();
            __syncthreads();
            if (tid == 0) st_release_sys(a.host_done + c, a.epoch);
        }
    }
    __threadfence_system();
}

// Per-stage constants: feasibility table, table tags, occupancy, what each profile can take and, for the rounds, the contention groups' spans
template <bool kSpec>
__device__ __forceinline__ void stage_init(const CandTab& tab, const PipeArgs& a, const Stage& st, PipeShared& s, SpecShared& ss) {
    const uint32_t tid = threadIdx.x;
    for (uint32_t i = tid; i < kSegMax * kSubMax / 4; i += kPipeThreads) st.occ32[i] = 0xFFFFFFFFu;
    for (uint32_t i = tid; i < kMaxTables * 256; i += kPipeThreads) s.feas[i] = a.feas[i];
    for (uint32_t i = tid; i < kSegMax * kSubMax; i += kPipeThreads) s.tab[i] = i < st.n_g ? a.gtab[st.lo + i] & (kMaxTables - 1) : 0;
    if (tid < ISL_MAX_PROFILES) {
        uint32_t n = 0, sz = 8;
        for (uint32_t k = 0; k < 4; ++k) for (uint32_t l = 0; l < 32; ++l) {
            const uint32_t d = tab.desc[k][l];
            if ((d >> 31) && (d & 15u) == tid) { ++n; sz = min(sz, (uint32_t)__popc((d >> 16) & 0xFFu)); }
        }
        s.maxacc[tid] = n;
        s.minsize[tid] = max(sz, 1u);           // smallest span of the profile over all tables
        const uint32_t have = __ballot_sync(0xFFFFu, n != 0);      // profiles that own at least one candidate: only these get a window
        if (n) s.plist[__popc(have & ((1u << tid) - 1u))] = tid;
        if (tid == 0) s.nplist = __popc(have);
    }
    if (tid >= 32 && tid < 32 + kMaxTables) {   // slices any candidate of the table can ever cover (REF_EXACT 80GB-class tables: 0x7F)
        uint32_t u = 0;
        for (uint32_t k = 0; k < 4; ++k) for (uint32_t l = 0; l < 32; ++l) {
            const uint32_t d = tab.desc[k][l];
            if ((d >> 31) && ((d >> 24) & 7u) == tid - 32) u |= (d >> 16) & 0xFFu;
        }
        s.usable[tid - 32] = u;
    }
    if (kSpec && tid >= 64 && tid < 96) {      // speculative rounds: the (profile, start) candidates of >= 4 slices as a list; per (table, profile) the slices of its smaller spans
        const uint32_t l = tid - 64;
        uint32_t n = 0;
        for (uint32_t k = 0; k < 4; ++k) {
            const uint32_t d = tab.desc[k][l];
            const bool big = (d >> 31) && __popc((d >> 16) & 0xFFu) >= 4;
            const uint32_t b = __ballot_sync(0xFFFFFFFFu, big);
            if (big) { const uint32_t at = n + __popc(b & ((1u << l) - 1u)); if (at < 32) ss.bigd[at] = d; }
            n += __popc(b);
        }
        if (l == 0) ss.nbigd = min(n, 32u);
        for (uint32_t i = l; i < kMaxTables * ISL_MAX_PROFILES; i += 32) {
            const uint32_t t = i / ISL_MAX_PROFILES, pp = i % ISL_MAX_PROFILES;
            uint32_t u = 0;
            for (uint32_t k = 0; k < 4; ++k) for (uint32_t x = 0; x < 32; ++x) {
                const uint32_t d = tab.desc[k][x];
                if ((d >> 31) && ((d >> 24) & 7u) == t && (d & 15u) == pp && __popc((d >> 16) & 0xFFu) < 4) u |= (d >> 16) & 0xFFu;
            }
            ss.smallm[t][pp] = (uint8_t)u;
        }
    }
    __syncthreads();
    for (uint32_t i = tid; i < st.n_g; i += kPipeThreads) reinterpret_cast<uint8_t*>(st.occ32)[i] = a.occ[st.lo + i];
    __syncthreads();
}

// The queues of a chunk (k_partition wrote them before this kernel started) are copied into shared memory with cp.async
// while the segment still waits for the chunk's token: they do not depend on the heads, so nothing is staged on the
// critical path between 'token in' and the first decision.  Offset -> thread mapping is the same for every chunk, so a
// thread's own wait_group orders its copies of consecutive chunks.
__device__ __forceinline__ void queue_load_async(const PipeArgs& a, const Stage& st, uint32_t chunk) {
    const char* src = reinterpret_cast<const char*>(a.q_all + (size_t)chunk * a.q_stride);
    const uint32_t bytes = (a.cctl[chunk].qoff[ISL_MAX_PROFILES] * 2u + 15u) & ~15u;
    for (uint32_t off = threadIdx.x * 16u; off < bytes; off += kPipeThreads * 16u)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(st.sa_q + off), "l"(src + off) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
}
// Fed streams: the requests of a batch may still be on their way (H2D + pre-pass on the feed stream) when the pipeline gets there.
// Causal window: chunk c additionally waits until every segment has committed chunk c - window; one deadline covers both waits.
// Returns true when the stream ends in front of this chunk (an open stream was closed, or the host aborted a feed).
__device__ __forceinline__ bool wait_ready(const PipeArgs& a, PipeShared& s, uint32_t chunk) {
    if (!a.ready && !a.window) return false;
    const bool gate_ring = a.ring_done && !a.inbox;          // ranks behind the owner are gated by the token itself
    if (threadIdx.x == 0) {
        bool closed = false;
        const unsigned long long t0 = globaltimer_ns();
        if (a.ready) {
            const uint32_t* f = a.ready + (a.open ? chunk : a.chunks[chunk].batch);
            // the feed kernels are launched AFTER this one; a tool that serialises kernels would starve the wait (the host side switches
            // feeding off when it detects one, ISL_NO_FEED=1 forces it) — fail loudly instead of hanging the GPU
            uint32_t v;
            wait_until([&] { v = ld_acquire_gpu(f); return v == a.epoch || v == ~a.epoch; }, a.wait_ns, 128, t0);
            closed = v == ~a.epoch;
        }
        if (!closed && a.window && chunk >= a.window) {
            if (gate_ring) wait_until([&] { return ld_acquire_sys(a.ring_done + chunk - a.window) >= a.world; }, a.wait_ns, 64, t0);
            else if (!a.ring_done) wait_until([&] { return ld_acquire_gpu(a.done_cnt + chunk - a.window) >= a.n_seg; }, a.wait_ns, 64, t0);
        }
        s.closed = closed;
    }
    __syncthreads();
    return s.closed != 0;
}
__device__ __forceinline__ void chunk_done(const PipeArgs& a, uint32_t chunk) {     // after the barrier that ends the chunk's commit
    if (a.done_cnt && threadIdx.x == 0) {
        if (a.ring_done) __threadfence_system(); else __threadfence();
        const uint32_t before = atomicAdd(a.done_cnt + chunk, 1u);
        if (a.ring_done && before + 1 == a.n_seg) atomicAdd_system(a.ring_done + chunk, 1u);     // this rank is through with the chunk
    }
}

// 1. frees of this batch inside my range: one byte per GPU
__device__ __forceinline__ void apply_frees(const PipeArgs& a, const Stage& st, const ChunkDesc& cd) {
    const uint8_t* fa = a.free_acc + (size_t)cd.batch * a.free_stride + st.lo;
    for (uint32_t i = threadIdx.x; i < st.n_g; i += kPipeThreads) {
        const uint32_t f = fa[i];
        if (f) atomicAnd(&st.occ32[i >> 2], ~(f << ((i & 3u) * 8u)));
    }
    __syncthreads();
}

// 2. local sweep: thread t owns kSegMax / kPipeThreads consecutive local GPUs; ordered compaction.  One scan carries both counts:
// candidates (low half) and free usable slices on the candidates (high half) — the latter bounds what the segment can accept: a profile
// of span z pops at most free / z requests here
__device__ __forceinline__ void sweep_subsegment(const Stage& st, PipeShared& s, uint32_t sb_base, uint32_t n_sb, uint32_t active) {
    constexpr uint32_t kGpt = kSegMax / kPipeThreads;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t og[kGpt], tg[kGpt];
    bool fg[kGpt];
    uint32_t cnt = 0;
#pragma unroll
    for (uint32_t x = 0; x < kGpt; ++x) {
        const uint32_t g = kGpt * tid + x;
        og[x] = reinterpret_cast<const uint8_t*>(st.occ32)[sb_base + g]; tg[x] = s.tab[sb_base + g];
        fg[x] = g < n_sb && (s.feas[tg[x] * 256 + og[x]] & active);
        if (fg[x]) cnt += 1u | ((uint32_t)__popc(~og[x] & s.usable[tg[x]]) << 16);
    }
    uint32_t incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += t; }
    if (lane == 31) s.warp[warp] = incl;
    __syncthreads();
    uint32_t off = incl - cnt;
    for (uint32_t x = 0; x < warp; ++x) off += s.warp[x];
    const uint32_t nfree = (off + cnt) >> 16;
    off &= 0xFFFFu;
#pragma unroll
    for (uint32_t x = 0; x < kGpt; ++x) if (fg[x]) st.cand[off++] = ((kGpt * tid + x) << 16) | table_tag(tg[x]) | og[x];
    if (tid == kPipeThreads - 1) { s.ncand = off; s.nfree = nfree; for (uint32_t x = 0; x < kCandPad; ++x) st.cand[off + x] = kInf; }   // sentinels: nothing fits
    __syncthreads();                    // s.ncand / s.nfree of the sweep are visible to warp 0
}

// Round 0 of the speculative rounds: what this stage's occupancy can take, per contention group -> predicted entry heads (ss.specH)
__device__ __forceinline__ void predict_entry(const PipeArgs& a, const Stage& st, PipeShared& s, SpecShared& ss, const Rounds& r,
                                              uint32_t c, uint32_t active, uint32_t sb_base, uint32_t n_sb) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, gseg = r.gseg;
    const Ctrl* cc = a.cctl + c;
    uint16_t* s_mj = reinterpret_cast<uint16_t*>(st.wkey);             // scratch (the windows are staged later): [3][kSpecStride] gathered masses of the stages in front
    if (tid < ISL_MAX_PROFILES) {
        const bool on = ((active >> tid) & 1u) && s.maxacc[tid] != 0 && cc->qcnt[tid] != 0;
        ss.qc[tid] = on ? cc->qcnt[tid] : 0u; ss.qo[tid] = cc->qoff[tid];
        const uint32_t big = __ballot_sync(0xFFFFu, on && s.minsize[tid] >= 4), small = __ballot_sync(0xFFFFu, on && s.minsize[tid] < 4);
        if (tid == 0) { ss.grp_big = big; ss.grp_small = small; ss.acc[0] = 0; ss.acc[1] = 0; ss.acc[2] = 0; }
        if (tid < kMaxTables) { uint32_t us = 0; for (uint32_t m = small; m; m &= m - 1) us |= ss.smallm[tid][__ffs(m) - 1]; ss.us[tid] = us; }   // slices the small group can use, per table
    }
    __syncthreads();
    {   // per GPU: the big group takes the widest span that still fits, twice at most (two quads); the small group fills the usable rest
        constexpr uint32_t kGpt = kSegMax / kPipeThreads;
        const uint32_t gb = ss.grp_big, nb = ss.nbigd;
        uint32_t mq = 0, mw = 0, mo = 0;
#pragma unroll
        for (uint32_t x = 0; x < kGpt; ++x) {
            const uint32_t g = kGpt * tid + x;
            if (g < n_sb) {
                const uint32_t t = s.tab[sb_base + g], o0 = reinterpret_cast<const uint8_t*>(st.occ32)[sb_base + g], us = ss.us[t];
                uint32_t o = o0;
                for (uint32_t it = 0; it < 2; ++it) {
                    uint32_t best = 0;
                    for (uint32_t y = 0; y < nb; ++y) {
                        const uint32_t d = ss.bigd[y], mk = (d >> 16) & 0xFFu;
                        if (((d >> 24) & 7u) == t && ((gb >> (d & 15u)) & 1u) && (o & mk) == 0 && __popc(mk) > __popc(best)) best = mk;
                    }
                    if (!best) break;
                    o |= best; ++mq;
                }
                mw += __popc(~o & us); mo += __popc(~o0 & us);
            }
        }
        mq = __reduce_add_sync(0xFFFFFFFFu, mq); mw = __reduce_add_sync(0xFFFFFFFFu, mw); mo = __reduce_add_sync(0xFFFFFFFFu, mo);
        if (lane == 0) { atomicAdd(&ss.acc[0], mq); atomicAdd(&ss.acc[1], mw); atomicAdd(&ss.acc[2], mo); }
    }
    __syncthreads();
    if (tid == 0) {
        spec_pub_down(a, r.sm.m + gseg * 2, r.tagb | ss.acc[0]);
        spec_pub_down(a, r.sm.m + gseg * 2 + 1, r.tagb | (min(ss.acc[1], 0xFFFFu) << 16) | min(ss.acc[2], 0xFFFFu));
    }
    if (tid < gseg) {       // masses of every stage in front of this one
        unsigned long long w0, w1;
        wait_until([&] {
            w0 = spec_ld(a, r.sm.m + tid * 2); w1 = spec_ld(a, r.sm.m + tid * 2 + 1);
            return (w0 >> 32) == (r.tagb >> 32) && (w1 >> 32) == (r.tagb >> 32);
        }, a.wait_ns, 0);
        s_mj[tid] = (uint16_t)w0; s_mj[kSpecStride + tid] = (uint16_t)(w1 >> 16); s_mj[2 * kSpecStride + tid] = (uint16_t)w1;
    }
    __syncthreads();
    if (tid < 32) {         // the big group takes its placements until its queues run dry; the small group fills what is left
        uint32_t totb = 0, tots = 0;
        for (uint32_t m = ss.grp_big; m; m &= m - 1) totb += ss.qc[__ffs(m) - 1];
        for (uint32_t m = ss.grp_small; m; m &= m - 1) { const uint32_t pp = __ffs(m) - 1; tots += ss.qc[pp] * s.minsize[pp]; }
        constexpr uint32_t kPer = (kSpecStride + 31) / 32;
        uint32_t ql = 0;
        for (uint32_t x = 0; x < kPer; ++x) { const uint32_t j = lane * kPer + x; if (j < gseg) ql += s_mj[j]; }
        uint32_t incl = ql;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += t; }
        uint32_t run = incl - ql, rr = 0;
        for (uint32_t x = 0; x < kPer; ++x) {
            const uint32_t j = lane * kPer + x;
            if (j < gseg) { rr += run < totb ? s_mj[kSpecStride + j] : s_mj[2 * kSpecStride + j]; run += s_mj[j]; }
        }
        rr = __reduce_add_sync(0xFFFFFFFFu, rr);
        const uint32_t Q = min(__shfl_sync(0xFFFFFFFFu, incl, 31), totb), R = min(rr, tots);
        const uint32_t hg = gseg > 0 ? shift_groups(0u, s, ss, (int)Q, (int)R, lane) : 0u;
        if (lane < ISL_MAX_PROFILES) ss.specH[lane] = hg;
    }
    __syncthreads();
}

// 3. entry heads (the token, the prediction or what the previous sub-segment left), window sizes and layout, the idle test and the
// cut-off of a speculative simulation.  Returns true when nothing placeable is pending at these heads.
template <bool kSpec>
__device__ __forceinline__ bool read_entry(const PipeArgs& a, const Stage& st, PipeShared& s, SpecShared& ss, uint32_t c, uint32_t sb,
                                           uint32_t active, bool known_exact, unsigned long long* tr, unsigned long long* dbg, uint32_t rnd) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, seg = st.seg;
    const size_t tok_chunk = (size_t)c * (a.n_seg + 1);
    asm volatile("cp.async.wait_group 0;" ::: "memory");       // my share of the chunk's queues has landed (long ago, as a rule)
    if (tid < 32) {
        uint32_t h = 0, wn = 0, left = 0;
        bool from_done = false;
        const uint32_t tag = token_tag(a);
        stamp_if(tr && tid == 0, tr + 0);
        if (kSpec) {                 // the predicted (or, at stage 0, the true) token
            if (tid < ISL_MAX_PROFILES) h = ss.specH[tid];
        } else if (sb > 0) {        // behind the first sub-segment the heads are the ones its chain left
            if (tid < ISL_MAX_PROFILES) h = s.heads[tid] + s.pop[tid];
        } else if (seg > 0) {
            // Token words are self-validating (token_tag): no separate flag, no fence on the producer side and no second round trip on this
            // side — lanes 0..15 each poll their own word of the previous segment's token or of the chunk's 'done' record (whichever is
            // valid first: when both are, they hold the same heads).  This poll is on every token hop and has no deadline: the stage in
            // front is itself in a wait that traps, or working.
            const uint32_t* pt = a.tokens + (tok_chunk + seg - 1) * kTokStride + (tid & 15u);
            const uint32_t* pd = a.tokens + (tok_chunk + a.n_seg) * kTokStride + (tid & 15u);
            bool ok = tid >= ISL_MAX_PROFILES;
            while (!__all_sync(0xFFFFFFFFu, ok)) {
                if (!ok) {
                    uint32_t v = ld_relaxed_gpu(pt);
                    if ((v >> 17) == tag) { h = v & 0x1FFFFu; ok = true; }
                    else { v = ld_relaxed_gpu(pd); if ((v >> 17) == tag) { h = v & 0x1FFFFu; ok = true; from_done = true; } }
                }
            }
        } else if (a.inbox) {       // first segment of a rank that has a predecessor: the token comes over NVLink
            // Every word is written with ONE relaxed system-scope store (4-byte stores are single-copy atomic): no fence and no flag on the
            // sender's side, one NVLink write latency per hop.  The consumer clears its slot after reading, so a tag can never be mistaken
            // for one of 32 768 streams ago.  A dead or stuck predecessor must not hang this GPU for good: the wait traps.
            uint32_t* slot = const_cast<uint32_t*>(a.inbox) + (size_t)c * kTokStride + (tid & 15u);
            const uint32_t xtag = xtoken_tag(a);
            bool ok = tid >= ISL_MAX_PROFILES;
            wait_until([&] {
                if (!ok) { const uint32_t v = ld_relaxed_sys(slot); if ((v >> 17) == xtag) { h = v & 0x1FFFFu; ok = true; } }
                return __all_sync(0xFFFFFFFFu, ok);
            }, a.wait_ns, 0);
            if (tid < ISL_MAX_PROFILES) st_relaxed_sys(slot, 0u);
        }
        stamp_if(tr && tid == 0, tr + 1);
        const bool all_done = sb == 0 && __all_sync(0xFFFFFFFFu, from_done || tid >= ISL_MAX_PROFILES);
        if (tid < ISL_MAX_PROFILES) {
            const Ctrl* cc = a.cctl + c;
            const uint32_t qc = kSpec ? ss.qc[tid] : cc->qcnt[tid], qo = kSpec ? ss.qo[tid] : cc->qoff[tid];     // re-simulations: no trip to L2
            left = ((active >> tid) & 1u) && qc > h ? qc - h : 0u;
            wn = min(left, min(s.ncand * s.maxacc[tid], s.nfree / s.minsize[tid]));   // no more pops than that are possible here
            s.heads[tid] = h; s.pop[tid] = 0;
            if (!kSpec) {
                s.wn[tid] = wn;
                s.qbeg[tid] = qo + h;                                       // first pending entry in the shared copy of the queues
            }
        }
        bool win_keep = true;
        if (kSpec) {
            // A corrected entry usually sits a few requests from the one simulated before: the windows are staged with kWinMargin entries on
            // either side and stay for the next simulation when every profile's new window [h, h + wn + 2) lies inside what is staged (real
            // keys behind the first wn entries are as good as the INF sentinels there: capacity, not the window, ends a profile's pops)
            uint32_t lo = 0, len = 0, woff = 0;
            bool ok = true;
            const uint32_t qc = tid < ISL_MAX_PROFILES ? ss.qc[tid] : 0u;
            if (tid < ISL_MAX_PROFILES) {
                lo = ss.wlo[tid]; len = ss.wlen[tid];
                if (left == 0) woff = len;                                  // nothing pending: straight onto the sentinels
                else { ok = ss.wvalid && h >= lo && (h + wn + 2 <= lo + len || lo + len >= qc); woff = h - lo; }
            }
            win_keep = __all_sync(0xFFFFFFFFu, ok);
            if (!win_keep && tid < ISL_MAX_PROFILES) {
                if (left == 0) { lo = h; len = 0; woff = 0; }
                else { lo = h - min(h, kWinMargin); len = min(qc - lo, (h - lo) + wn + kWinMargin + 2); woff = h - lo; }
                ss.wlo[tid] = lo; ss.wlen[tid] = len;
                s.qbeg[tid] = ss.qo[tid] + lo;
            }
            if (tid < ISL_MAX_PROFILES) { ss.woff[tid] = woff; s.wn[tid] = len - woff; }     // real entries from the entry to the staged end
            wn = len;                                                       // the layout below counts the staged entries
        }
        // nothing placeable is pending any more: tell every later segment at once instead of relaying hop by hop
        const bool idle = __ballot_sync(0xFFFFFFFFu, left != 0) == 0;
        if (idle && !all_done && !kSpec && tid < ISL_MAX_PROFILES) st_relaxed_gpu(a.tokens + (tok_chunk + a.n_seg) * kTokStride + tid, tag_word(tag, h));
        if (tid == 0) {
            s.idle = idle ? 1u : 0u;
            if (kSpec) {        // an idle simulation stages nothing: a new layout that was never filled must not be kept by the next one
                ss.restage = win_keep ? 0u : 1u;
                if (!win_keep) ss.wvalid = idle ? 0u : 1u;
                // A speculative simulation from an entry that is far off can run several times longer than the segment's true work (everything
                // the stages in front are wrongly believed to have left over lands here) and would hold up the whole round.  Unless the entry
                // is known to be the true one, the simulation is cut off at 1.3 x the largest complete one so far; a cut-off round publishes
                // the exit extrapolated from the last complete simulation instead (what the stages behind would assume anyway).
                s.cap = ss.capst[1] && !known_exact ? min(kLogCap + 1, ((ss.capst[0] * 21u) >> 4) + 64u) : kLogCap + 1;
                ss.capped = 0;
            } else s.cap = kLogCap + 1;
        }
        uint32_t incl = wn + kWinPad;                       // INF sentinels close every window
#pragma unroll
        for (int d = 1; d < 16; d <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, incl, d); if ((int)lane >= d) incl += t; }
        if (tid < ISL_MAX_PROFILES) s.wbase[tid] = incl - (wn + kWinPad);
    }
    __syncthreads();
    stamp_if(tr && tid == 0, tr + 8);
    stamp_if(dbg && tid == 0, dbg + rnd * 8 + 1);
    return s.idle != 0;
}

// Windows of ready-made keys t << 15 | profile << 11, each closed by two INF sentinels — converted from the shared copy of the queues
// (a shared-memory round trip per round instead of an L2 one), only for profiles that own candidates
template <bool kSpec>
__device__ __forceinline__ void stage_windows(const Stage& st, PipeShared& s, const SpecShared& ss, unsigned long long* tr) {
    const uint32_t tid = threadIdx.x;
    const uint32_t npl = kSpec && !ss.restage ? 0u : s.nplist;
    for (uint32_t x = 0; x < npl; ++x) {
        const uint32_t p = s.plist[x], wn = kSpec ? ss.wlen[p] : s.wn[p], pk = p << 11, qb = s.qbeg[p];
        uint32_t* __restrict__ dst = st.wkey + s.wbase[p];
        // plain, unconditional (clamped) accesses: the loads of a round overlap instead of queueing behind each other
        for (uint32_t i = tid; i < wn + kWinPad; i += kPipeThreads) { const uint32_t v = st.q[qb + min(i, wn)]; dst[i] = i < wn ? (v << 15) | pk : kInf; }
    }
    stamp_if(tr && tid == 0, tr + 10);
    store_if(tr && tid == 0, tr + 11, s.wn[s.plist[0]] | ((unsigned long long)s.nfree << 32));
    __syncthreads();
    stamp_if(tr && tid == 0, tr + 9);
}

// 4. the decision chain (see k_chain), tuned for the shortest loop-carried path, and 5. the token for the next segment behind the
// stage's last sub-segment.  By the chain warp.
template <int K, bool kP15, bool kSpec>
__device__ __forceinline__ void decide(const PipeArgs& a, const Stage& st, PipeShared& s, SpecShared& ss, const ChainSlots<K>& cs, PipeCounters& n,
                                       uint32_t c, bool last_sub, unsigned long long* tr, unsigned long long* dbg, uint32_t rnd) {
    const uint32_t lane = threadIdx.x & 31u, sa_cand = st.sa_cand, sa_log = st.sa_log;
    const uint32_t *cmask = cs.cmask, *klow = cs.klow, *cprof = cs.cprof, n_cand = s.ncand;
    uint32_t tcur[K], tnext[K], tnn[K], wa[K], wa0[K];
    const uint32_t* wnp[K];         // &s.wn of each slot's profile, formed once: computed next to s.wbase inside the loop it slowed the rounds
#pragma unroll
    for (int k = 0; k < K; ++k) {
        wa0[k] = st.sa_wkey + 4 * (s.wbase[cprof[k]] + (kSpec ? ss.woff[cprof[k]] : 0u));
        const bool has = cs.valid[k];
        tcur[k] = has ? lds_u32(wa0[k]) | klow[k] : kInf;               // INF | anything = INF
        tnext[k] = has ? lds_u32(wa0[k] + 4) | klow[k] : kInf;
        wnp[k] = s.wn + cprof[k];
        const bool two = has && *wnp[k] >= 1;                           // a third entry exists only behind >= 1 real one
        tnn[k] = two ? lds_u32(wa0[k] + 8) : kInf;
        wa[k] = wa0[k] + 12;                                            // next entry to load on a pop
    }
    uint32_t la = sa_log, ca = sa_cand + 8;                             // ca: shared address of candidate record (current + 2)
    // Per slot the loop carries conflict words z = occupancy & candidate mask of the current / next / next-but-one candidate GPU
    // and g = "fits on that GPU ? sel bit : nothing" as a ready OR mask; the key of the NEXT decision is formed at the end of the
    // body.  Loop-carried path behind the redux: sign mask of `sel` -> bitwise mux of z -> fold the winner's slices in and test
    // (one LOP3 with a predicate output) -> pick the key: four ALU levels (a freshly updated occupancy register tested through
    // ISETP / SEL needs five, and ISETP + SEL behind the redux is the slower of the two: tools/microbench_pred.cu times both).
    // The updates are issued unconditionally and the "nothing fits" test comes LAST: a branch is not speculated, so a test in
    // front of the updates would put its resolution on the loop-carried path of every decision.  m == INF behaves like a decision
    // that lands on the next GPU and pops only exhausted lanes (no real key has all-ones t / profile fields unless profile 15
    // is in use, kP15); the rare path rewinds the cursors and reloads the conflict words after the jump.
    uint32_t z0[K], z1[K], z2[K], g1[K], g2[K], cm8[K];
    auto reload_z = [&]() {
        const uint32_t a0 = lds_u16(ca - 8), a1 = lds_u16(ca - 4), a2 = lds_u16(ca);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            z0[k] = a0 & cmask[k]; z1[k] = a1 & cmask[k]; z2[k] = a2 & cmask[k];
            g1[k] = z1[k] == 0 ? 0x80000000u : kInf; g2[k] = z2[k] == 0 ? 0x80000000u : kInf;
        }
    };
#pragma unroll
    for (int k = 0; k < K; ++k) cm8[k] = cmask[k] & 0xFFu;
    reload_z();
    uint32_t key = kInf, a2 = lds_u16(ca);
    auto first_key = [&]() {
        key = kInf;
#pragma unroll
        for (int k = 0; k < K; ++k) key = min(key, z0[k] == 0 ? tcur[k] : (tcur[k] | g1[k]));
    };
    first_key();
    const unsigned long long jumps0 = n.jumps;
    // (trace stamps next to the decision loop perturb its schedule in the instantiation with the rounds and slow every round; that
    // instantiation records its cell at certification instead)
    if (!kSpec) stamp_if(tr && lane == 0, tr + 4);
    stamp_if(dbg && lane == 0, dbg + rnd * 8 + 2);
    constexpr bool kDefer = !kP15;      // the "nothing fits" test runs once per unrolled group, not per decision; see the rare path below
    const uint32_t la_cap = sa_log + 8u * s.cap;
    bool cut = false;
    while (true) {
        if (!kDefer && la >= la_cap) { cut = true; break; }     // once per group of decisions, off the loop-carried path
        bool none = false;
        uint32_t m = 0, mmax = 0;
        uint32_t lm[kUnroll], lc[kUnroll];     // kDefer: the group's log records, stored behind its last decision
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {     // unrolled: one taken branch per kUnroll decisions
            m = redux_min_u32(key);
#pragma unroll
            for (int k = 0; k < K; ++k) {       // in the shadow of the redux: the record fetched by the previous decision (the same one again if it did not advance)
                z2[k] = a2 & cmask[k];
                g2[k] = z2[k] == 0 ? 0x80000000u : kInf;
            }
            if (kP15) { none = m == kInf; if (none) break; }
            uint32_t ks;
            asm("shr.s32 %0, %1, 31;" : "=r"(ks) : "r"(m));                                            // all ones: landed on the next GPU
            asm("mad.lo.s32 %0, %1, -4, %0;" : "+r"(ca) : "r"(ks));                                     // ca += sel * 4
            if (kDefer) {
                lm[u] = m; lc[u] = ca;
                mmax = max(mmax, m);
            } else {
                sts_v2_if(lane == 0, la, m, ca);                // decision log: (key, address of the record two past the GPU it landed on)
                la += 8;
            }
            a2 = lds_u16(ca);
            key = kInf;
#pragma unroll
            for (int k = 0; k < K; ++k) {
                const bool adv = kP15 ? (((m & 0x7FFFF800u) ^ tcur[k]) & 0xFFFFF800u) == 0 : ((m ^ tcur[k]) & 0x7FFFF800u) == 0;
                const uint32_t tn = adv ? tnext[k] : tcur[k];
                uint32_t zs, gn, kk;
                asm("lop3.b32 %0, %1, %2, %3, 0xca;" : "=r"(zs) : "r"(ks), "r"(z1[k]), "r"(z0[k]));       // sel ? z1 : z0
                asm("lop3.b32 %0, %1, %2, %3, 0xca;" : "=r"(gn) : "r"(ks), "r"(g2[k]), "r"(g1[k]));       // sel ? g2 : g1
                asm("{ .reg .pred p; lop3.b32 %1, %2, %3, %4, 0xF8; setp.eq.u32 p, %1, 0; selp.b32 %0, %5, %6, p; }"     // z0 = zs | winner's slices
                    : "=r"(kk), "=r"(z0[k]) : "r"(zs), "r"(m), "r"(cm8[k]), "r"(tn), "r"(tn | gn));
                key = min(key, kk);
                g1[k] = gn;
                asm("lop3.b32 %0, %1, %2, %3, 0xca;" : "=r"(z1[k]) : "r"(ks), "r"(z2[k]), "r"(z1[k]));    // sel ? z2 : z1
                tcur[k] = tn;
                tnext[k] = adv ? (tnn[k] | klow[k]) : tnext[k];
                tnn[k] = lds_u32_if(adv, wa[k], tnn[k]);        // consumed at the earliest one pop later
                wa[k] = add_if(adv, wa[k], 4u);
            }
            if (!kP15 && !kDefer) {
                none = m == kInf;
                if (__builtin_expect(none, 0)) {
                    ca -= 4; la -= 8;                           // rewind the pseudo-decision
#pragma unroll
                    for (int k = 0; k < K; ++k)
                        if (tcur[k] == kInf) { tnext[k] = kInf; wa[k] -= 4; }
                    break;
                }
            }
        }
        uint32_t from = (ca - sa_cand) >> 2;        // record index of (current + 2)
        if (kDefer) {
            // m == INF is a legitimate step of the recurrence ("neither this GPU nor the next takes anything: the next one becomes
            // current"; it pops only lanes whose window is exhausted, into their INF sentinels), so the loop body needs no exit
            // test per decision — one test per group: did ANY decision of the group find nothing?
            // The group's log is written here, behind its last decision: a store between two reductions (with its predicate, and the
            // address update that waits until the store has read its registers) would sit on the in-order issue path of every decision.
            if (__builtin_expect(mmax != kInf, 1)) {
                // every decision real: eight stores at fixed offsets, by all lanes (the same record; a lane predicate here is
                // compiled into a branch around each store)
#pragma unroll
                for (int u = 0; u < kUnroll; ++u) sts_v2_if(true, la + 8u * u, lm[u], lc[u]);
                la += 8u * kUnroll;
                if (__builtin_expect(la < la_cap, 1)) continue;     // (the cut-off test rides on the group's one branch)
                cut = true; break;
            }
            // a pseudo-decision (m == INF: nothing fits here or on the next GPU, move on by one) leaves no log record
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const bool real = lm[u] != kInf;
                sts_v2_if(lane == 0 && real, la, lm[u], lc[u]);
                la = add_if(real, la, 8u);
            }
            if (la >= la_cap) { cut = true; break; }
            // exhausted lanes were popped past the end of their windows: back onto the sentinels (at most kUnroll pops since the last time)
#pragma unroll
            for (int k = 0; k < K; ++k)
                if (tcur[k] == kInf) { tnext[k] = kInf; tnn[k] = kInf; wa[k] = wa0[k] + 12 + 4 * *wnp[k]; }
            if (m != kInf) continue;                // the group ended on a real decision: carry on
            from -= 1;                              // the pseudo-decision already moved on by one GPU: the new 'next' is still unexamined
        } else if (__builtin_expect(!none, 1)) continue;
        uint32_t alive = 0;
#pragma unroll
        for (int k = 0; k < K; ++k) alive |= tcur[k] != kInf ? 1u << cprof[k] : 0u;
        const uint32_t j = pipeline_skip(sa_cand, s.feas, n_cand, from, alive, lane);
        ++n.jumps;
        if (j == kInf) break;
        ca = sa_cand + 4 * (j + 2);
        reload_z();
        a2 = lds_u16(ca);
        first_key();
    }
    const uint32_t nlog = (la - sa_log) >> 3;
    if (!kSpec) {
        stamp_if(tr && lane == 0, tr + 5);
        stamp_if(dbg && lane == 0, dbg + rnd * 8 + 3);
        store_if(tr && lane == 0, tr + 6, nlog);
        store_if(tr && lane == 0, tr + 7, (n.jumps - jumps0) | ((unsigned long long)(((ca - sa_cand) >> 2) - 2) << 32));
        n.steps += nlog; n.visited += ((ca - sa_cand) >> 2) - 2;
    } else {
        n.spec_steps = nlog; n.spec_visited = ((ca - sa_cand) >> 2) - 2; ++n.sims;
    }
#pragma unroll
    for (int k = 0; k < K; ++k) if (cs.reports[k]) s.pop[cprof[k]] = min((wa[k] - wa0[k] - 12) >> 2, *wnp[k]);
    __syncwarp();
    if (last_sub && lane < ISL_MAX_PROFILES && !kSpec) publish_token(a, c, st.seg, lane, s.heads[lane] + s.pop[lane]);    // the next segment starts
    __syncwarp();
    if (lane == 0) {
        s.nlog = nlog;
        if (kSpec) ss.capped = cut ? 1u : 0u;
        if (tr) tr[2] = globaltimer_ns();
    }
}

// The round's exchange: publish exit heads X and consumed masses D, read the predecessor's X and every earlier stage's D, then certify
// (returns true: the log in shared memory is THE log) or correct the predicted entry for the next round
__device__ __forceinline__ bool exchange_round(const PipeArgs& a, uint32_t seg, PipeShared& s, SpecShared& ss, Rounds& r, PipeCounters& n,
                                               uint32_t c, unsigned long long* tr, unsigned long long* dbg) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, rnd = r.rnd, gseg = r.gseg;
    const unsigned long long tagr = r.tagb | ((unsigned long long)rnd << 32);
    if (tid < 32) {
        uint32_t X = 0, dq, dr, pop = 0;
        const bool was_cut = ss.capped != 0;
        if (tid < ISL_MAX_PROFILES) { pop = s.pop[tid]; X = s.heads[tid] + pop; }
        if (was_cut) {      // exit of the last complete simulation, moved by what the entry has moved since (per group, shares as always)
            uint32_t eq, er;
            group_masses(tid < ISL_MAX_PROFILES ? s.heads[tid] - ss.Hc[tid] : 0u, s, ss, lane, eq, er);
            const uint32_t xe = shift_groups(tid < ISL_MAX_PROFILES ? ss.Xc[tid] : 0u, s, ss, (int)eq, (int)er, lane);
            if (tid < ISL_MAX_PROFILES) { X = max(xe, s.heads[tid]); pop = X - s.heads[tid]; }
        }
        if (tid < ISL_MAX_PROFILES) { ss.specX[tid] = X; if (!was_cut) { ss.Hc[tid] = s.heads[tid]; ss.Xc[tid] = X; } }
        if (tid == 0) { if (was_cut) ss.capst[2] = 0; else { ss.capst[0] = max(ss.capst[0], s.nlog); ss.capst[1] = 1; ss.capst[2] = 1; } }
        group_masses(pop, s, ss, lane, dq, dr);
        if (rnd >= 3 && gseg + 1 < r.gtot && !(r.need_sim && !s.idle)) wait_ack(a, r);     // (checked behind the chain when one ran)
        if (tid < ISL_MAX_PROFILES) spec_pub_nb(a, seg, r.sm.x + ((size_t)gseg * 2 + (rnd & 1u)) * 16 + tid, tagr | X, false);
        if (tid == 16) spec_pub_down(a, r.sm.d + (size_t)rnd * kSpecStride + gseg, tagr | ((r.c_prev ? 1u : 0u) << 31) | (dq << 13) | dr);
        if (tid == 0) { ss.dqr[0] = dq; ss.dqr[1] = dr; ss.acc[0] = 0; ss.acc[1] = 0; }
        stamp_if(dbg && tid == 0, dbg + rnd * 8 + 4);
    }
    __syncthreads();
    bool cbit = true;
    if (tid < gseg) {       // D of every stage in front
        const unsigned long long w = read_record(a, r.sm.d + (size_t)rnd * kSpecStride + tid, r.sm.df + tid, tagr, r);
        cbit = r.p_final || ((w >> 31) & 1u);
        atomicAdd(&ss.acc[0], (uint32_t)(w >> 13) & 0x7FFu);
        atomicAdd(&ss.acc[1], (uint32_t)w & 0x1FFFu);
    }
    if (gseg > 0 && tid >= 192 && tid < 192 + ISL_MAX_PROFILES) {      // X of the stage in front
        const uint32_t i = tid - 192;
        ss.specXp[i] = (uint32_t)read_record(a, r.sm.x + ((size_t)(gseg - 1) * 2 + (rnd & 1u)) * 16 + i, r.sm.xf + (size_t)(gseg - 1) * 16 + i, tagr, r) & 0x1FFFFu;
    }
    if (tid + 1 == gseg) ss.predc = cbit ? 1u : 0u;         // the bit of the stage right in front of me
    const int unset = __syncthreads_count(!cbit);
    const bool allc = unset == 0;
    // Knowledge lags a round: the stage whose entry becomes the true one NEXT round sits behind a consistent prefix whose last member's
    // bit is not set yet (that member's own entry became the true one only this round).  So "everything in front but the stage right
    // in front of me is consistent" already exempts the next simulation from the cut-off — otherwise the frontier itself could be cut
    // off and every step of it would cost a second round (tests/spec_rounds_model.cpp).
    const bool near = allc || (unset == 1 && !ss.predc);
    const bool certified = allc && r.c_prev;
    stamp_if(dbg && tid == 0, dbg + rnd * 8 + 5);
    store_if(dbg && tid == 0, dbg + rnd * 8 + 7, s.nlog | ((unsigned long long)r.need_sim << 32));
    if (gseg > 0 && tid == 192) spec_pub_nb(a, seg, r.sm.ack + gseg, ((unsigned long long)r.tage << 32) | (certified ? 0xFFFFu : rnd), true);
    if (certified) {    // every entry up to mine was the true token one round ago and has not moved since
        if (tid < ISL_MAX_PROFILES) spec_pub_nb(a, seg, r.sm.xf + (size_t)gseg * 16 + tid, r.tagF | (rnd << 24) | ss.specX[tid], false);
        if (tid == 16) spec_pub_down(a, r.sm.df + gseg, r.tagF | (rnd << 24) | (ss.dqr[0] << 13) | ss.dqr[1]);
        if (tid == 0) {
            n.steps += n.spec_steps; n.visited += n.spec_visited;
            if (gseg == r.gtot - 1) { n.rounds_sum += rnd; ++n.cells; }
            if (tr) { tr[0] = r.t_cell; tr[2] = globaltimer_ns(); tr[6] = s.nlog; tr[7] = n.sims - r.sims_cell; tr[11] = rnd; }
        }
        return true;
    }
    if (tid < 32) {     // c for the next round; the corrected prediction
        const bool same = tid >= ISL_MAX_PROFILES || ss.specH[tid] == ss.specXp[tid];
        const bool cnow = __all_sync(0xFFFFFFFFu, same);
        const uint32_t hold = tid < ISL_MAX_PROFILES ? ss.specH[tid] : 0u;
        uint32_t hn = tid < ISL_MAX_PROFILES ? ss.specXp[tid] : 0u, mq, mr;
        group_masses(hn, s, ss, lane, mq, mr);
        hn = shift_groups(hn, s, ss, (int)ss.acc[0] - (int)mq, (int)ss.acc[1] - (int)mr, lane);
        {   // Two candidates for the next entry: the Newton step (hn) and plain chaining (the exit of the stage in front as it is).  Where a
            // batch's contested front reaches far the Newton step over-corrects round after round; each stage uses the rule whose
            // candidate of the PREVIOUS round came closer to what the stage in front has published now (study, section 8).
            const uint32_t xp = tid < ISL_MAX_PROFILES ? ss.specXp[tid] : 0u;
            uint32_t ea = 0, eb = 0;
            if (tid < ISL_MAX_PROFILES && ss.havepred) { ea = (uint32_t)abs((int)ss.predA[tid] - (int)xp); eb = (uint32_t)abs((int)ss.predB[tid] - (int)xp); }
            ea = __reduce_add_sync(0xFFFFFFFFu, ea); eb = __reduce_add_sync(0xFFFFFFFFu, eb);
            __syncwarp();
            if (tid < ISL_MAX_PROFILES) { ss.predA[tid] = hn; ss.predB[tid] = xp; }
            if (tid == 0) ss.havepred = 1;
            if (eb < ea) hn = xp;
        }
        if (tid < ISL_MAX_PROFILES) ss.specH[tid] = hn;
        const bool moved = tid < ISL_MAX_PROFILES && hn != hold;
        const bool changed = __any_sync(0xFFFFFFFFu, moved);
        // a cut-off simulation left no usable log: the entry is simulated again (in full once it is known to be the true one) and counts as
        // inconsistent until then
        if (tid == 0) ss.specflag = (cnow && ss.capst[2] ? 1u : 0u) | (changed || !ss.capst[2] ? 2u : 0u);
        stamp_if(dbg && tid == 0, dbg + rnd * 8 + 6);
    }
    __syncthreads();
    r.c_prev = ss.specflag & 1u; r.need_sim = ss.specflag & 2u; r.known_exact = near;
    if (++r.rnd >= kSpecRounds - 1) __trap();      // cannot happen: every round certifies at least one more stage
    return false;
}

// 6. commit: result records + occupancy bits of the logged decisions
__device__ __forceinline__ void commit_log(const PipeArgs& a, const Stage& st, const PipeShared& s, const ChunkDesc& cd, uint32_t sb_base,
                                           unsigned long long* tr) {
    const uint32_t nlog = s.nlog;
    for (uint32_t j = threadIdx.x; j < nlog; j += kPipeThreads) {
        const uint2 e = st.log[j];
        const uint32_t l = sb_base + (st.cand[((e.y - st.sa_cand) >> 2) - 2] >> 16), mask = e.x & 0xFFu, t = (e.x >> 15) & 0xFFFFu;
        const uint2 rec = pack_result(flip_gpu(st.lo + l, a.flip), __ffs(mask) - 1, __popc(mask), ISL_ST_PLACED);
        a.out[cd.req_off + t] = rec;
        if (a.owner_out) a.owner_out[cd.req_off + t] = rec;         // partitioned inventory: straight into the owner rank's result array (peer store over NVLink)
        atomicOr(&st.occ32[l >> 2], mask << ((l & 3u) * 8u));
    }
    __syncthreads();
    if (tr && threadIdx.x == 0) tr[3] = globaltimer_ns();
}

// 3.-5. through the plain pipeline.  Returns false when nothing placeable is pending at the entry: the token went on unchanged, and the
// stage's remaining sub-segments have nothing to take either.
template <int K, bool kP15>
__device__ __forceinline__ bool resolve_plain(const PipeArgs& a, const Stage& st, PipeShared& s, SpecShared& ss, const ChainSlots<K>& cs,
                                              PipeCounters& n, uint32_t c, uint32_t sb, uint32_t active, bool last_sub, unsigned long long* tr) {
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (read_entry<false>(a, st, s, ss, c, sb, active, false, tr, nullptr, 1)) {
        if (warp == 0) {    // pass-through: the token (unchanged heads) still reaches the next rank / the caller from the last segment
            if (lane < ISL_MAX_PROFILES) publish_token(a, c, st.seg, lane, s.heads[lane]);
            __syncwarp();
            if (lane == 0 && tr) { tr[2] = globaltimer_ns(); tr[3] = tr[2]; }
        }
        __syncthreads();
        return false;
    }
    stage_windows<false>(st, s, ss, tr);
    if (is_chain_warp(warp)) decide<K, kP15, false>(a, st, s, ss, cs, n, c, last_sub, tr, nullptr, 1);
    __syncthreads();
    return true;
}

// 3.-5. by speculative rounds (one sub-segment per stage): predict the entry, then simulate, exchange and correct round by round until
// the stage is certified
template <int K, bool kP15>
__device__ __forceinline__ void resolve_rounds(const PipeArgs& a, const Stage& st, PipeShared& s, SpecShared& ss, const ChainSlots<K>& cs,
                                               PipeCounters& n, uint32_t c, uint32_t active, uint32_t sb_base, uint32_t n_sb, unsigned long long* tr) {
    const uint32_t tid = threadIdx.x;
    Rounds r;
    r.sm = spec_mem(a.spec_mem, c);
    r.tage = a.spec_world > 1 ? a.xepoch : a.epoch;        // a partitioned inventory tags with the stream id all ranks share
    r.tagb = (unsigned long long)((r.tage & 0xFFFFFFu) << 8) << 32; r.tagF = r.tagb | (0xFFull << 32);
    r.gseg = a.spec_base + st.seg; r.gtot = a.spec_total;
    predict_entry(a, st, s, ss, r, c, active, sb_base, n_sb);
    // known_exact: everything in front of the stage right in front of me was consistent one round ago: my next entry may be the true one
    r.rnd = 1; r.c_prev = r.gseg == 0; r.need_sim = true; r.known_exact = r.gseg == 0; r.p_final = false; r.p_word = 0;
    if (tid == 0) { ss.capst[0] = 0; ss.capst[1] = 0; ss.capst[2] = 0; s.cap = kLogCap + 1; ss.capped = 0; ss.wvalid = 0; ss.havepred = 0; }
    r.t_cell = tr ? globaltimer_ns() : 0ull; r.sims_cell = n.sims;
#ifdef ISL_SPEC_DBG_STAMPS      // per-round stamps of one cell (tools/spec_trace.py): a debugging build — the extra live pointer around the decision loop slows it
    unsigned long long* dbg = a.spec_dbg && a.spec_dbg_cell == ((c << 16) | st.seg) ? a.spec_dbg : nullptr;
#else
    constexpr unsigned long long* dbg = nullptr;
#endif
    do {
        stamp_if(dbg && tid == 0, dbg + r.rnd * 8 + 0);
        if (r.need_sim) {       // an unchanged entry is not simulated again
            if (read_entry<true>(a, st, s, ss, c, 0, active, r.known_exact, tr, dbg, r.rnd)) {
                if (tid == 0) { s.nlog = 0; n.spec_steps = 0; n.spec_visited = 0; }    // nothing pending at these heads: the exit equals the entry
            } else {
                stage_windows<true>(st, s, ss, tr);
                if (is_chain_warp(tid >> 5)) decide<K, kP15, true>(a, st, s, ss, cs, n, c, true, tr, dbg, r.rnd);
                else if (tid == kPipeThreads - 32 && r.rnd >= 3 && r.gseg + 1 < r.gtot) wait_ack(a, r);     // in the shadow of the chain
            }
            __syncthreads();
        }
    } while (!exchange_round(a, st.seg, s, ss, r, n, c, tr, dbg));
}

template <int K, bool kP15, bool kSpec>
__global__ void __launch_bounds__(kPipeThreads, 1) k_pipeline(CandTab tab, PipeArgs a) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ PipeShared s;
    __shared__ SpecShared ss;
    const uint32_t tid = threadIdx.x, seg = blockIdx.x;
    if (seg == a.n_seg) { deliver_chunks(a); return; }
    Stage st;
    st.seg = seg; st.lo = min(a.hi, a.lo + seg * a.seg); st.n_g = min(a.hi, st.lo + a.seg) - st.lo;
    st.occ32 = reinterpret_cast<uint32_t*>(smem); st.cand = reinterpret_cast<uint32_t*>(smem + kPipeOffCand); st.log = reinterpret_cast<uint2*>(smem + kPipeOffLog);
    st.q = reinterpret_cast<const uint16_t*>(smem + kPipeOffQ); st.wkey = reinterpret_cast<uint32_t*>(smem + kPipeOffWin);
    st.sa_cand = (uint32_t)__cvta_generic_to_shared(st.cand); st.sa_log = (uint32_t)__cvta_generic_to_shared(st.log);
    st.sa_q = (uint32_t)__cvta_generic_to_shared(st.q); st.sa_wkey = (uint32_t)__cvta_generic_to_shared(st.wkey);
    stage_init<kSpec>(tab, a, st, s, ss);
    const ChainSlots<K> cs(tab, tid & 31u);
    PipeCounters n{};

    bool closed = wait_ready(a, s, 0);
    if (!closed) queue_load_async(a, st, 0);
    for (uint32_t c = 0; c < a.n_chunks && !closed; ++c) {
        const ChunkDesc cd = a.chunks[c];
        if (cd.first_of_batch) apply_frees(a, st, cd);
        const uint32_t active = a.cctl[c].active;
        // A stage is walked sub-segment by sub-segment (one for inventories up to SMs x 512 GPUs): sweep, heads, windows, chain, commit per
        // sub-segment; the token is awaited in front of the first and published behind the last one (or as soon as nothing is pending).
        const uint32_t n_sub = max(1u, (st.n_g + a.sub - 1) / a.sub);
        bool prefetched = false;            // the next chunk's queues are on their way (they may only overwrite this chunk's after its last chain)
        for (uint32_t sb = 0; sb < n_sub; ++sb) {
            const uint32_t sb_base = sb * a.sub, n_sb = min(a.sub, st.n_g - min(st.n_g, sb_base));
            const bool last_sub = sb + 1 == n_sub;
            unsigned long long* tr = a.trace ? a.trace + ((size_t)c * a.n_seg + seg) * kTraceWords : nullptr;
            sweep_subsegment(st, s, sb_base, n_sb, active);
            // kSpec (host: only with one sub-segment per stage) is a separate instantiation, so that the plain pipeline's code is untouched by the rounds' machinery
            if (kSpec) resolve_rounds<K, kP15>(a, st, s, ss, cs, n, c, active, sb_base, n_sb, tr);
            else if (!resolve_plain<K, kP15>(a, st, s, ss, cs, n, c, sb, active, last_sub, tr)) break;
            if (last_sub && c + 1 < a.n_chunks && !a.ready && !a.window) { queue_load_async(a, st, c + 1); prefetched = true; }   // the chain is done with the queues: fetch the next chunk's behind the commit
            commit_log(a, st, s, cd, sb_base, tr);
        }
        chunk_done(a, c);
        if (c + 1 < a.n_chunks && !prefetched) { closed = wait_ready(a, s, c + 1); if (!closed) queue_load_async(a, st, c + 1); }   // fed / windowed stream: the next batch may not be due yet
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    for (uint32_t i = tid; i < st.n_g; i += kPipeThreads) a.occ[st.lo + i] = reinterpret_cast<uint8_t*>(st.occ32)[i];
    if (a.owner_out) __threadfence_system();        // the peer stores of this CTA are performed before the grid is seen as complete
    if (tid == 0 && n.steps + n.jumps) {
        atomicAdd(&a.stats->placed, n.steps);
        atomicAdd(&a.stats->steps, n.steps);
        atomicAdd(&a.stats->visited, n.visited);
        atomicAdd(&a.stats->jumps, n.jumps);
    }
    if (kSpec && tid == 0) {
        atomicAdd(&a.stats->spec_sims, n.sims);
        atomicAdd(&a.stats->spec_rounds, n.rounds_sum);
        atomicAdd(&a.stats->spec_cells, (unsigned long long)n.cells);
    }
}

// ---------------------------------------------------------------------------------------------
// k_capacity: the what-if / defragmentation query (SURVEY 8f-4).  cap[p] = how many more pods of profile p ALONE the GPUs of [lo, hi)
// could still take = sum over GPUs of capn[table][p][occupancy] (the same per-byte table the scan-mode commit places from).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_capacity(const uint8_t* __restrict__ occ, const uint8_t* __restrict__ gtab, const uint8_t* __restrict__ capn,
                                                   uint32_t n_profiles, uint32_t lo, uint32_t hi, unsigned long long* __restrict__ cap) {
    __shared__ unsigned long long s_cap[ISL_MAX_PROFILES];
    if (threadIdx.x < ISL_MAX_PROFILES) s_cap[threadIdx.x] = 0;
    __syncthreads();
    uint32_t acc[ISL_MAX_PROFILES];
#pragma unroll
    for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) acc[p] = 0;
    for (uint32_t g = lo + blockIdx.x * blockDim.x + threadIdx.x; g < hi; g += gridDim.x * blockDim.x) {
        const uint32_t o = occ[g], t = gtab[g] & (kMaxTables - 1);
#pragma unroll
        for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) if (p < n_profiles) acc[p] += capn[(t * ISL_MAX_PROFILES + p) * 256 + o];
    }
#pragma unroll
    for (uint32_t p = 0; p < ISL_MAX_PROFILES; ++p) {
        uint32_t v = acc[p];
#pragma unroll
        for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, d);
        if ((threadIdx.x & 31u) == 0 && v) atomicAdd(&s_cap[p], (unsigned long long)v);
    }
    __syncthreads();
    if (threadIdx.x < ISL_MAX_PROFILES && s_cap[threadIdx.x]) atomicAdd(&cap[threadIdx.x], s_cap[threadIdx.x]);
}

// ---------------------------------------------------------------------------------------------
// k_bestfit: ISL_POLICY_BEST_FIT (extension, SURVEY 8a-ext — no reference counterpart, parity is against
// oracle/ref_fast.cpp's best-fit).  Among the GPUs on which the profile has a legal start, take the one with the
// fewest free slices after the placement = the highest popcount of the occupancy byte, ties to the lowest canonical
// index; the start is the reference's first legal start.  Requests are resolved strictly in order (request-major: a
// placement can make a GPU the best fit of the very next request, so there is no GPU-major shortcut).
// State: GPUs grouped by occupancy byte (256 classes); per class a two-level bitmap (32 GPUs per word, 1024 per
// summary bit) and its minimum member.  One warp: lane = a few classes, key = (8 - popcount) << 24 | class minimum,
// redux.min picks the GPU; lane 0 moves it to its new class.  One CTA; all threads build the class structure.
// kGang (isl_place_gangs): the requests come in gangs [gang_off[i], gang_off[i + 1]) that commit all or nothing.  With a zero score table
// (ISL_POLICY_FIRST_FIT / _RIGHT_TO_LEFT) the key is the class minimum, i.e. exact first-fit.  The first ALLOC of a gang that cannot be
// placed keeps its record, the gang's later members are not tried, and when the gang ends its placed members are moved back to their old
// classes in reverse order (a PLACED record holds gpu, start and size: `occupancy & ~span` is the byte it came from) and, like every
// other ALLOC of the gang, reported GANG_ABORTED.  The `dead` profile mask assumes occupancy only grows: it is restored as well, except
// for a profile that died before any member of its gang was placed (it died in the committed state).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kBfThreads = 1024;
constexpr uint32_t kBfMaxGpus = 1u << 20;           // class bitmaps: G / 32 words + G / 1024 summary words per (table, occupancy byte) class
constexpr uint32_t kBfSmemGpus = 4096;              // up to here the class bitmaps live in shared memory (132 KiB)

template <bool kMulti, bool kGang = false>
__global__ void __launch_bounds__(kBfThreads, 1) k_bestfit(uint32_t n, const uint2* __restrict__ in, uint2* __restrict__ out, uint8_t* __restrict__ occ,
                                                           uint32_t lo, uint32_t hi, const uint8_t* __restrict__ lut, DevProfiles prof,
                                                           uint32_t* __restrict__ g_bitmaps, Ctrl* ctrl, const uint8_t* __restrict__ score,
                                                           const uint8_t* __restrict__ gtab, const uint8_t* __restrict__ sizes, uint32_t n_tables,
                                                           const uint32_t* __restrict__ gang_off = nullptr, uint32_t n_gangs = 0) {
    extern __shared__ __align__(16) uint32_t s_dyn[];
    // a class = (table of the GPU's node, occupancy byte): every GPU of a class behaves the same for every profile
    __shared__ uint32_t s_min[kMaxTables * 256];
    __shared__ uint8_t s_lut[ISL_MAX_PROFILES * 256];
    // what the policy minimises, per (table, profile, occupancy byte): ISL_POLICY_BEST_FIT = free slices (8 - popcount), ISL_POLICY_MIN_FRAG =
    // (profile, start) pairs of the table that stop being feasible when the profile takes its first legal start there (host-built)
    __shared__ uint8_t s_score[ISL_MAX_PROFILES * 256];
    __shared__ uint8_t s_sizes[kMaxTables * ISL_MAX_PROFILES];
    const uint32_t tid = threadIdx.x, lane = tid & 31u;
    const uint32_t Gr = hi - lo, W0 = (Gr + 31) / 32, W1 = (W0 + 31) / 32, stride = W0 + W1;   // words per class
    const uint32_t n_cls = n_tables * 256;
    const bool small = n_tables == 1 && Gr <= kBfSmemGpus;      // bitmaps in shared memory; otherwise in global memory, zeroed by the host
    uint32_t* bm = small ? s_dyn : g_bitmaps;
    if (small) for (uint32_t i = tid; i < 256 * stride; i += kBfThreads) bm[i] = 0;
    // one table (kMulti == false): the per-byte tables sit in shared memory; several: they are read from global memory (L1-resident,
    // 8 KiB per table)
    if (!kMulti) for (uint32_t i = tid; i < ISL_MAX_PROFILES * 256; i += kBfThreads) { s_lut[i] = lut[i]; s_score[i] = score[i]; }
    auto lut_at = [&](uint32_t idx) -> uint32_t { return kMulti ? (uint32_t)__ldg(lut + idx) : (uint32_t)s_lut[idx]; };
    auto score_at = [&](uint32_t idx) -> uint32_t { return kMulti ? (uint32_t)__ldg(score + idx) : (uint32_t)s_score[idx]; };
    if (tid < kMaxTables * ISL_MAX_PROFILES) s_sizes[tid] = sizes[tid];
    for (uint32_t i = tid; i < n_cls; i += kBfThreads) s_min[i] = kInf;
    __syncthreads();
    for (uint32_t g = tid; g < Gr; g += kBfThreads) {           // build: every GPU joins its class
        const uint32_t c = (kMulti ? (uint32_t)(gtab[lo + g] & (kMaxTables - 1)) * 256u : 0u) + occ[lo + g];
        atomicOr(&bm[c * stride + (g >> 5)], 1u << (g & 31u));
        atomicOr(&bm[c * stride + W0 + (g >> 10)], 1u << ((g >> 5) & 31u));
        atomicMin(&s_min[c], g);
    }
    __syncthreads();
    if (!is_chain_warp(tid >> 5)) return;
    // lane 0: GPU g leaves the class whose bitmaps are c0 and joins the one of c1 (independent words, loads first)
    auto move_bits = [&](uint32_t* c0, uint32_t* c1, uint32_t g) {
        const uint32_t w0 = c0[g >> 5] & ~(1u << (g & 31u)), w1 = c1[g >> 5] | (1u << (g & 31u));
        const uint32_t s1 = c1[W0 + (g >> 10)] | (1u << ((g >> 5) & 31u));
        c0[g >> 5] = w0; c1[g >> 5] = w1; c1[W0 + (g >> 10)] = s1;
        if (w0 == 0) c0[W0 + (g >> 10)] &= ~(1u << ((g >> 5) & 31u));
    };
    // new minimum of the class of c0 after its minimum g left it (nothing below g).  Usually it sits under the summary word that held g:
    // every lane reads that word (one broadcast); only when it is empty do the lanes look at the further summary words, 32 at a time
    auto min_after = [&](const uint32_t* c0, uint32_t g) -> uint32_t {
        uint32_t mn = kInf;
        const uint32_t k = g >> 10, sw = c0[W0 + k];
        if (sw) { const uint32_t wi = k * 32 + __ffs(sw) - 1; mn = wi * 32 + __ffs(c0[wi]) - 1; }
        else
            for (uint32_t k0 = k + 1; k0 < W1; k0 += 32) {
                const uint32_t s2 = k0 + lane < W1 ? c0[W0 + k0 + lane] : 0u;
                const uint32_t b = __ballot_sync(0xFFFFFFFFu, s2 != 0);
                if (b) {
                    const uint32_t src = __ffs(b) - 1;
                    const uint32_t wi = (k0 + src) * 32 + __ffs(__shfl_sync(0xFFFFFFFFu, s2, src)) - 1;
                    mn = wi * 32 + __ffs(c0[wi]) - 1;
                    break;
                }
            }
        return mn;
    };
    uint32_t placed = 0;
    uint32_t dead = 0;              // profiles that found no GPU: occupancy only grows inside a batch's ALLOC phase, so they never will again
    // kGang: the open gang is requests [g_first, g_end); g_fail = its member that could not be placed (kInf: none yet); g_placed = its
    // members placed so far; dead_at = `dead` when it began.  Lane l holds gang_off[g_win + 1 + l]: one load per 32 gangs
    uint32_t gang = 0, g_first = 0, g_end = 0, g_fail = kInf, g_placed = 0, dead_at = 0, g_win = 0, g_offs = 0;
    if (kGang) {
        g_offs = lane < n_gangs ? __ldg(gang_off + 1 + lane) : n;
        g_end = __shfl_sync(0xFFFFFFFFu, g_offs, 0);
    }
    // kGang, the open gang failed: its placed members (every ALLOC before g_fail) leave their classes again, last placed first, and
    // report GANG_ABORTED (the members after g_fail already do)
    auto abort_gang = [&]() {
        for (uint32_t top = g_fail; g_placed;) {
            const uint32_t cnt = min(32u, top - g_first), r = top - 1 - lane;       // lane order = descending request order
            const uint2 q = lane < cnt ? in[r] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
            const bool alloc = ((q.y >> 8) & 0xFFu) == ISL_OP_ALLOC;
            const uint2 rec = alloc ? out[r] : make_uint2(0, 0);
            uint32_t undo = __ballot_sync(0xFFFFFFFFu, alloc);
            while (undo) {
                const uint32_t src = __ffs(undo) - 1;
                undo &= undo - 1;
                const uint32_t rx = __shfl_sync(0xFFFFFFFFu, rec.x, src), ry = __shfl_sync(0xFFFFFFFFu, rec.y, src);
                const uint32_t p = __shfl_sync(0xFFFFFFFFu, q.y, src) & 0xFFu;
                const uint32_t g = flip_gpu(rx, prof.flip) - lo, span = slice_span(ry & 0xFFu, (ry >> 8) & 0xFFu);
                const uint32_t t = kMulti ? (uint32_t)(gtab[lo + g] & (kMaxTables - 1)) : 0u;
                const uint32_t o2 = occ[lo + g], cw2 = (t << 8) | o2, cw = (t << 8) | (o2 & ~span);
                uint32_t* c2 = bm + cw2 * stride;
                const bool was_min = s_min[cw2] == g;
                __syncwarp();
                if (lane == 0) {                                // back from class o2 to class o2 & ~span
                    move_bits(c2, bm + cw * stride, g);
                    occ[lo + g] = (uint8_t)(o2 & ~span);
                    out[top - 1 - src] = pack_result(ISL_GPU_NONE, ISL_START_NONE, prof.rows[p].size, ISL_ST_GANG_ABORTED);
                    if (g < s_min[cw]) s_min[cw] = g;
                    --placed;
                }
                __syncwarp();
                if (was_min) {
                    const uint32_t mn = min_after(c2, g);
                    if (lane == 0) s_min[cw2] = mn;
                }
                __syncwarp();
                --g_placed;
            }
            top -= cnt;
        }
        dead = dead_at;
    };
    // kGang: end every gang that lies wholly before request `upto` (commit, or abort when a member failed)
    auto close_gangs = [&](uint32_t upto) {
        while (g_end <= upto && gang < n_gangs) {
            if (g_fail != kInf) abort_gang();
            g_fail = kInf; g_placed = 0; dead_at = dead; g_first = g_end;
            if (++gang < n_gangs) {
                if (gang - g_win == 32) { g_win = gang; g_offs = gang + lane < n_gangs ? __ldg(gang_off + gang + 1 + lane) : n; }
                g_end = __shfl_sync(0xFFFFFFFFu, g_offs, gang - g_win);
            }
        }
    };
    uint2 ahead = lane < n ? in[lane] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
    for (uint32_t base = 0; base < n; base += 32) {
        const uint2 mine = ahead;                               // the next block's requests are fetched while this one is resolved
        ahead = base + 32 + lane < n ? in[base + 32 + lane] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
        // only the live ALLOCs of the block are looked at (frees, unknown or dead profiles: defaults were written by k_prepare); in a
        // gang every ALLOC is looked at, since an unknown or dead profile fails its gang
        uint32_t live;
        {
            const uint32_t wp = mine.y & 0xFFu, wop = (mine.y >> 8) & 0xFFu;
            live = __ballot_sync(0xFFFFFFFFu, wop == ISL_OP_ALLOC && (kGang || (wp < prof.n && !((dead >> wp) & 1u))));
        }
        while (live) {
            const uint32_t j = __ffs(live) - 1;
            live &= live - 1;
            const uint32_t p = __shfl_sync(0xFFFFFFFFu, mine.y, j) & 0xFFu;
            if (kGang) {
                close_gangs(base + j);
                if (g_fail != kInf) {                           // a member of this gang failed: the rest is not tried
                    if (lane == 0) out[base + j] = pack_result(ISL_GPU_NONE, ISL_START_NONE, p < prof.n ? prof.rows[p].size : 0u, ISL_ST_GANG_ABORTED);
                    continue;
                }
                if (p >= prof.n || ((dead >> p) & 1u)) { g_fail = base + j; continue; }
            } else if ((dead >> p) & 1u) continue;              // died inside this block
            uint32_t key = kInf, kc = 0;
#pragma unroll 8
            for (uint32_t c = lane; c < n_cls; c += 32) {       // lane l looks at classes l, l+32, ...
                const uint32_t mn = s_min[c];
                const uint32_t idx = ((c >> 8) * ISL_MAX_PROFILES + p) * 256 + (c & 255u);
                if (mn != kInf && lut_at(idx) != ISL_START_NONE) {
                    const uint32_t k2 = (score_at(idx) << 24) | mn;
                    if (k2 < key) { key = k2; kc = c; }
                }
            }
            const uint32_t m = __reduce_min_sync(0xFFFFFFFFu, key);
            if (m == kInf) {                                    // stays NO_CAPACITY, and so does every later request of the profile
                dead |= 1u << p;
                if (kGang) {
                    g_fail = base + j;
                    if (g_placed == 0) dead_at |= 1u << p;      // nothing of the gang placed yet: it died in the committed state
                }
                continue;
            }
            const uint32_t g = m & 0xFFFFFFu;
            const uint32_t cw = __shfl_sync(0xFFFFFFFFu, kc, __ffs(__ballot_sync(0xFFFFFFFFu, key == m)) - 1);   // the class IS (table, occupancy byte)
            const uint32_t t = cw >> 8, o = cw & 255u;
            const uint32_t start = lut_at((t * ISL_MAX_PROFILES + p) * 256 + o), size = s_sizes[t * ISL_MAX_PROFILES + p];
            const uint32_t o2 = o | slice_span(start, size), cw2 = (t << 8) | o2;
            uint32_t* c0 = bm + cw * stride;
            uint32_t* c1 = bm + cw2 * stride;
            __syncwarp();                                       // all lanes have read the class minima before they are rewritten
            if (lane == 0) {                                    // the GPU leaves class o and joins class o2
                move_bits(c0, c1, g);
                occ[lo + g] = (uint8_t)o2;
                out[base + j] = pack_result(flip_gpu(lo + g, prof.flip), start, size, ISL_ST_PLACED);
                if (g < s_min[cw2]) s_min[cw2] = g;
                ++placed;
            }
            if (kGang) ++g_placed;
            __syncwarp();
            const uint32_t mn = min_after(c0, g);               // g was the class minimum
            if (lane == 0) s_min[cw] = mn;
            __syncwarp();
        }
    }
    if (kGang) close_gangs(n);
    if (lane == 0) count_placed(ctrl, placed);
}

// ---------------------------------------------------------------------------------------------
// Priority preemption (isl_preempt, DESIGN.md 4.7).
//   k_victim_map  one thread per victim: validates its span and claims its slices in the per-slice victim-index map (partition-local
//                 GPU x 8 words, kVictimNone where no listed victim covers the slice); any violation raises a bit of *err
//   k_preempt     one cooperative launch for the whole call: each CTA keeps its contiguous share of the partition in shared memory,
//                 every preemptor is one 64-bit min over all (GPU, legal start) candidates (grid_min)
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kVictimNone = 0xFFFFFFFFu;
constexpr uint32_t kPreThreads = 512;
constexpr uint32_t kPreMaxGpus = 1u << 20;              // the key's GPU field has 24 bits; the gang limit of the engine's other paths
// Shared memory per GPU of a CTA's share: 8 priority bytes, the occupancy byte, the run-start byte, the table byte.  At kPreMaxGpus over
// the 132 SMs of an H100 a CTA holds 7 944 GPUs = 87 KB, below the 227 KB a CTA may opt into on sm_90 (the host checks the device's limit).
constexpr uint32_t kPreBytesPerGpu = 11;
constexpr uint32_t kVmErrSpan = 1u, kVmErrFree = 2u, kVmErrOverlap = 4u;

__global__ void k_victim_map(uint32_t n, const isl_victim* __restrict__ victims, const uint8_t* __restrict__ occ, uint32_t G, uint32_t lo,
                             uint32_t hi, uint32_t flip, uint32_t* __restrict__ vmap, uint32_t* __restrict__ err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const isl_victim v = victims[i];
    if (v.gpu >= G || v.size == 0 || v.start + v.size > ISL_SLOTS) { atomicOr(err, kVmErrSpan); return; }
    const uint32_t gi = flip_gpu(v.gpu, flip);
    if (gi < lo || gi >= hi) return;                    // outside the partition: ignored, as isl_free_batch ignores such spans
    const uint32_t span = slice_span(v.start, v.size);   // start + size <= 8: the cut changes nothing
    if ((occ[gi] & span) != span) atomicOr(err, kVmErrFree);
    uint32_t* w = vmap + (size_t)(gi - lo) * ISL_SLOTS;
    for (uint32_t s = v.start; s < v.start + v.size; ++s)
        if (atomicCAS(w + s, kVictimNone, i) != kVictimNone) atomicOr(err, kVmErrOverlap);
}

struct PreemptArgs {            // kernel parameter (by value)
    const uint2* in;            // requests (isl_request)
    const uint8_t* prio;        // priority of every request
    const isl_victim* victims;
    const uint32_t* vmap;       // k_victim_map's output
    const uint8_t* occ;         // the live occupancy (storage order), read only
    const uint8_t* gtab;        // table of every GPU's node (storage order)
    const uint8_t* masks;       // [table][profile][position in the row]: candidate_mask of that start, 0 = none
    uint2* out;
    uint32_t* evict;            // n x 8 victim indices
    unsigned long long* keys;   // [2][gridDim.x] per-CTA minima, double-buffered by preemptor parity
    uint32_t n, lo, Gr, per_cta;
};

// Candidate key, lexicographic (isl_preempt rule 5):  [50:42] highest priority in V + 1, 0 for an empty V | [41:31] sum of V's
// priorities (<= 8 x 254) | [30:27] |V| | [26:3] GPU in scan order (partition-local storage index) | [2:0] position of the start in the
// row.  V of a legal (GPU, start) is every victim that overlaps the mask: one head slice per victim — the run starts inside the mask, plus
// the mask's lowest slice when it is busy (a victim that begins below the mask).
__device__ __forceinline__ unsigned long long preempt_key(uint32_t m, uint32_t o, uint32_t rs, unsigned long long pr, uint32_t g, uint32_t k) {
    const uint32_t heads = (rs & m) | (o & m & (m & (0u - m)));
    uint32_t mx = 0, sum = 0;
    for (uint32_t h = heads; h; h &= h - 1) {
        const uint32_t b = (uint32_t)(pr >> (8 * (__ffs(h) - 1))) & 0xFFu;
        mx = max(mx, b + 1u); sum += b;
    }
    return ((unsigned long long)mx << 42) | ((unsigned long long)sum << 31) | ((unsigned long long)__popc(heads) << 27) |
           ((unsigned long long)g << 3) | k;
}

__device__ __forceinline__ uint32_t warp_min(uint32_t v) { return redux_min_u32(v); }
__device__ __forceinline__ unsigned long long warp_min(unsigned long long v) {
    const uint32_t hi = redux_min_u32((uint32_t)(v >> 32));
    const uint32_t lo = redux_min_u32((uint32_t)(v >> 32) == hi ? (uint32_t)v : kInf);
    return ((unsigned long long)hi << 32) | lo;
}

// The minimum of `v` over every thread of a cooperative launch of kThreads threads per CTA, returned to every thread (k_preempt,
// k_ganglocal; DESIGN.md 4.7).  Every thread of every CTA must call it: it holds the grid barrier.  Each CTA reduces by warp,
// then across the block, and writes its minimum to keys[parity * gridDim.x + blockIdx.x]; after grid.sync warp 0 reads every CTA's
// minimum with __ldcg (other SMs wrote them; L1 is not coherent) and broadcasts the result through s_win.  The minima are double-buffered
// by `parity`, which the call flips: a fast CTA may write round i + 1 before a slow one has read round i.
template <uint32_t kThreads, typename T>
__device__ __forceinline__ T grid_min(T v, unsigned long long* keys, uint32_t& parity, T* s_warp, T* s_win) {
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    v = warp_min(v);
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = warp_min(lane < kThreads / 32 ? s_warp[lane] : ~T(0));
        if (lane == 0) keys[parity * gridDim.x + blockIdx.x] = v;
    }
    cooperative_groups::grid_group grid = cooperative_groups::this_grid();
    grid.sync();
    if (warp == 0) {
        v = ~T(0);
        for (uint32_t c = lane; c < gridDim.x; c += 32) v = min(v, (T)__ldcg(keys + parity * gridDim.x + c));
        v = warp_min(v);
        if (lane == 0) *s_win = v;
    }
    __syncthreads();
    parity ^= 1u;
    return *s_win;
}

__global__ void __launch_bounds__(kPreThreads, 1) k_preempt(PreemptArgs a, DevProfiles prof) {
    extern __shared__ __align__(8) unsigned char pre_smem[];
    __shared__ uint8_t s_masks[kMaxTables * ISL_MAX_PROFILES * ISL_MAX_STARTS];
    __shared__ unsigned long long s_warp[kPreThreads / 32];
    __shared__ unsigned long long s_win;
    const uint32_t tid = threadIdx.x;
    const uint32_t base = blockIdx.x * a.per_cta, cnt = base < a.Gr ? min(a.per_cta, a.Gr - base) : 0u;
    unsigned long long* s_prio = reinterpret_cast<unsigned long long*>(pre_smem);      // byte s = priority of slice s, 255 = no victim
    uint8_t* s_occ = pre_smem + (size_t)a.per_cta * 8;
    uint8_t* s_rs = s_occ + a.per_cta;                  // bit s: a victim begins at slice s
    uint8_t* s_tab = s_rs + a.per_cta;
    for (uint32_t i = tid; i < sizeof(s_masks); i += kPreThreads) s_masks[i] = a.masks[i];
    for (uint32_t g = tid; g < cnt; g += kPreThreads) {
        const uint4* w4 = reinterpret_cast<const uint4*>(a.vmap + (size_t)(base + g) * ISL_SLOTS);
        const uint4 w0 = w4[0], w1 = w4[1];
        const uint32_t w[ISL_SLOTS] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        unsigned long long pr = 0;
        uint32_t rs = 0;
#pragma unroll
        for (uint32_t s = 0; s < ISL_SLOTS; ++s) {
            const uint32_t p = w[s] == kVictimNone ? 0xFFu : a.victims[w[s]].priority;
            pr |= (unsigned long long)p << (8 * s);
            if (w[s] != kVictimNone && (s == 0 || w[s - 1] != w[s])) rs |= 1u << s;
        }
        s_prio[g] = pr; s_rs[g] = (uint8_t)rs;
        s_occ[g] = a.occ[a.lo + base + g]; s_tab[g] = a.gtab[a.lo + base + g];
    }
    __syncthreads();
    auto unplaced = [&](uint32_t i, uint32_t size, uint32_t status) {
        if (blockIdx.x == 0 && tid < ISL_SLOTS) {
            if (tid == 0) a.out[i] = pack_result(ISL_GPU_NONE, ISL_START_NONE, size, status);
            a.evict[(size_t)i * ISL_SLOTS + tid] = kVictimNone;
        }
    };
    uint32_t parity = 0;
    for (uint32_t i = 0; i < a.n; ++i) {
        const uint2 rq = a.in[i];
        const uint32_t profile = rq.y & 0xFFu, op = (rq.y >> 8) & 0xFFu;
        if (op != ISL_OP_ALLOC || profile >= prof.n) {      // the same for every CTA: no exchange
            unplaced(i, 0, op == ISL_OP_ALLOC ? ISL_ST_BAD_PROFILE : ISL_ST_NOOP);
            continue;
        }
        const uint32_t pi = a.prio[i];
        unsigned long long best = ~0ull;
        for (uint32_t g = tid; g < cnt; g += kPreThreads) {
            const unsigned long long pr = s_prio[g];
            const uint32_t o = s_occ[g], rs = s_rs[g];
            uint32_t ev = 0;                                // slices whose victim has a priority below the preemptor's
#pragma unroll
            for (uint32_t s = 0; s < ISL_SLOTS; ++s) ev |= (((uint32_t)(pr >> (8 * s)) & 0xFFu) < pi) << s;
            const uint32_t blocked = o & ~ev;
            const uint8_t* mk = s_masks + ((uint32_t)s_tab[g] * ISL_MAX_PROFILES + profile) * ISL_MAX_STARTS;
#pragma unroll
            for (uint32_t k = 0; k < ISL_MAX_STARTS; ++k) {
                const uint32_t m = mk[k];
                if (m && !(m & blocked)) best = min(best, preempt_key(m, o, rs, pr, base + g, k));
            }
        }
        const unsigned long long win = grid_min<kPreThreads>(best, a.keys, parity, s_warp, &s_win);
        if (win == ~0ull) { unplaced(i, prof.rows[profile].size, ISL_ST_NO_CAPACITY); continue; }     // no candidate anywhere
        const uint32_t gw = (uint32_t)(win >> 3) & 0xFFFFFFu, k = (uint32_t)win & 7u;
        if (gw - base < cnt && tid == 0) {                  // the CTA that owns the GPU applies the eviction to its own state
            const uint32_t g = gw - base, o = s_occ[g], rs = s_rs[g];
            const uint32_t m = s_masks[((uint32_t)s_tab[g] * ISL_MAX_PROFILES + profile) * ISL_MAX_STARTS + k];
            const uint32_t heads = (rs & m) | (o & m & (m & (0u - m)));
            const uint4* w4 = reinterpret_cast<const uint4*>(a.vmap + (size_t)gw * ISL_SLOTS);
            const uint4 w0 = w4[0], w1 = w4[1];
            const uint32_t w[ISL_SLOTS] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
            uint32_t idx[ISL_SLOTS], nv = 0, gone = 0;
            for (uint32_t h = heads; h; h &= h - 1) {
                const uint32_t v = w[__ffs(h) - 1];     // a victim leaves whole: every slice it covers is still its own
                uint32_t j = nv++;
                for (; j > 0 && idx[j - 1] > v; --j) idx[j] = idx[j - 1];
                idx[j] = v;
#pragma unroll
                for (uint32_t s = 0; s < ISL_SLOTS; ++s) gone |= (w[s] == v) << s;
            }
            const uint32_t touched = gone | m;          // freed or taken: either way no victim any more
            unsigned long long pr = s_prio[g];
#pragma unroll
            for (uint32_t s = 0; s < ISL_SLOTS; ++s) if ((touched >> s) & 1u) pr |= 0xFFull << (8 * s);
            s_prio[g] = pr; s_rs[g] = (uint8_t)(rs & ~touched); s_occ[g] = (uint8_t)((o & ~gone) | m);
            a.out[i] = pack_result(flip_gpu(a.lo + gw, prof.flip), __ffs(m) - 1, __popc(m), ISL_ST_PLACED);
            for (uint32_t j = 0; j < ISL_SLOTS; ++j) a.evict[(size_t)i * ISL_SLOTS + j] = j < nv ? idx[j] : kVictimNone;
        }
        __syncthreads();                                    // the owner's state is updated before its threads score the next preemptor
    }
}

// ---------------------------------------------------------------------------------------------
// k_nodefit: ISL_POLICY_MOST_ALLOCATED / ISL_POLICY_LEAST_ALLOCATED (DESIGN.md 4.8), the kube-scheduler's NodeResourcesFit scores over
// the nodes of the range, in MIG memory slices.  Request-major like k_bestfit: one placement changes one node's score, and the very next
// request sees it.  One CTA, one launch per batch behind k_prepare (frees and default records).
//   build    one thread per node: cap = width(table) x GPUs in range, busy = popcount of the occupancy under the width, and per profile
//            the GPUs that admit it; then per profile a 32-ary min-tree over the nodes, leaf key (100 - score) << 24 | local node index
//            (INF where the profile fits on none of the node's GPUs), so the root is the winning node with ties to the lowest index
//   request  every warp reads the root of the profile's tree.  INF: the default NO_CAPACITY record stands, the profile is dead for the
//            rest of the batch (occupancy only grows).  Otherwise the chain warp takes the node's first admitting GPU (32 per ballot) and
//            commits it; after a barrier warp q recounts profile q's fits on that node, rewrites its leaf and walks up (32 siblings and
//            one redux.min per level, stopping where a parent keeps its value); a second barrier ends the request.
// The trees live in shared memory up to kNfSmemNodes nodes and in global memory (L2) beyond.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kNfThreads = 32 * ISL_MAX_PROFILES;   // one warp per profile
constexpr uint32_t kNfSmemNodes = 2048;                  // up to here the trees live in shared memory (16 x 2 176 words = 136 KiB)
constexpr uint32_t kNfMaxNodes = 1u << 20;              // isl_load_inventory's limit for node scoring: empty nodes count, so not kBfMaxGpus
constexpr uint32_t kNfMaxLevels = 5;                     // 32^4 leaves >= kNfMaxNodes nodes
static_assert((1ull << (5 * (kNfMaxLevels - 1))) >= kNfMaxNodes, "a range of kNfMaxNodes nodes needs more tree levels");

struct NodeFitArgs {            // kernel parameter (by value)
    const uint2* in;
    uint2* out;
    uint8_t* occ;
    const uint8_t* gtab;        // table of every GPU's node
    const uint8_t* lut;         // [table][profile][occ]
    const uint8_t* sizes;       // [table][profile]
    const uint32_t* node_off;   // the inventory's node offsets (n_nodes + 1)
    uint32_t* tree;             // global trees ([profile][T] words), when they do not fit in shared memory
    uint32_t* fit;              // [profile][Nr]: GPUs of the node that admit the profile
    uint32_t* busy;             // [Nr]: busy slices under the width
    uint32_t* meta;             // [Nr]: cap | table << 24
    Ctrl* ctrl;
    uint32_t n, lo, hi, nlo, Nr;        // requests; the range; its first node and node count
    uint32_t most;                      // 1: MostAllocated, 0: LeastAllocated
    uint32_t levels, T;                 // tree levels (the last holds the root) and words per profile
    uint32_t lvl_off[kNfMaxLevels];     // first word of every level inside a profile's tree; level k has lvl_cnt[k] keys, padded to 32
    uint32_t lvl_cnt[kNfMaxLevels];
    uint8_t width[kMaxTables];          // largest start + size over the rows of every table
};

// The leaf key of a node for one profile: NodeResourcesFit's integer score with MaxNodeScore 100, smaller key = better node
__device__ __forceinline__ uint32_t nodefit_leaf(uint32_t fit, uint32_t busy, uint32_t cap, uint32_t req, uint32_t most, uint32_t node) {
    if (fit == 0) return kInf;
    const uint32_t score = most ? 100u * (busy + req) / cap : 100u * (cap - busy - req) / cap;
    return ((100u - score) << 24) | node;
}

__global__ void __launch_bounds__(kNfThreads, 1) k_nodefit(NodeFitArgs a, uint32_t n_profiles) {
    extern __shared__ __align__(16) uint32_t s_tree[];
    __shared__ uint8_t s_lut[kMaxTables * ISL_MAX_PROFILES * 256];
    __shared__ uint8_t s_sizes[kMaxTables * ISL_MAX_PROFILES];
    __shared__ uint32_t s_ev[2];                         // the committed GPU's occupancy byte before and after the request
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    uint32_t* tree = a.Nr <= kNfSmemNodes ? s_tree : a.tree;
    for (uint32_t i = tid; i < sizeof(s_lut) / 4; i += kNfThreads) reinterpret_cast<uint32_t*>(s_lut)[i] = reinterpret_cast<const uint32_t*>(a.lut)[i];
    if (tid < kMaxTables * ISL_MAX_PROFILES) s_sizes[tid] = a.sizes[tid];
    __syncthreads();
    auto admits = [&](uint32_t t, uint32_t q, uint32_t o) -> uint32_t { return s_lut[(t * ISL_MAX_PROFILES + q) * 256 + o] != ISL_START_NONE; };
    // build: one thread per node
    for (uint32_t v = tid; v < a.Nr; v += kNfThreads) {
        const uint32_t g0 = max(a.lo, __ldg(a.node_off + a.nlo + v)), g1 = min(a.hi, __ldg(a.node_off + a.nlo + v + 1));
        const uint32_t cnt = g1 > g0 ? g1 - g0 : 0u, t = cnt ? (uint32_t)(a.gtab[g0] & (kMaxTables - 1)) : 0u;
        const uint32_t wm = (1u << a.width[t]) - 1u, cap = a.width[t] * cnt;
        uint32_t busy = 0, fit[ISL_MAX_PROFILES] = {};
        for (uint32_t g = g0; g < g1; ++g) {
            const uint32_t o = a.occ[g];
            busy += __popc(o & wm);
#pragma unroll
            for (uint32_t q = 0; q < ISL_MAX_PROFILES; ++q) fit[q] += admits(t, q, o);
        }
        a.busy[v] = busy; a.meta[v] = cap | (t << 24);
#pragma unroll
        for (uint32_t q = 0; q < ISL_MAX_PROFILES; ++q)
            if (q < n_profiles) {
                a.fit[(size_t)q * a.Nr + v] = fit[q];
                tree[(size_t)q * a.T + v] = nodefit_leaf(fit[q], busy, cap, s_sizes[t * ISL_MAX_PROFILES + q], a.most, v);
            }
    }
    for (uint32_t k = 0; k < a.levels; ++k) {            // level k from level k - 1 (leaves: only their padding), padding INF
        __syncthreads();
        const uint32_t cnt = a.lvl_cnt[k], padded = (cnt + 31u) & ~31u;
        for (uint32_t i = tid; i < n_profiles * padded; i += kNfThreads) {
            const uint32_t q = i / padded, j = i - q * padded;
            uint32_t* lv = tree + (size_t)q * a.T + a.lvl_off[k];
            if (j >= cnt) lv[j] = kInf;
            else if (k > 0) {
                const uint32_t* below = tree + (size_t)q * a.T + a.lvl_off[k - 1];
                uint32_t m = kInf;
                for (uint32_t c = 0; c < 32; ++c) m = min(m, below[j * 32 + c]);
                lv[j] = m;
            }
        }
    }
    __syncthreads();
    const uint32_t root = a.lvl_off[a.levels - 1];
    uint32_t placed = 0, dead = 0;
    uint2 ahead = lane < a.n ? a.in[lane] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
    for (uint32_t base = 0; base < a.n; base += 32) {
        const uint2 mine = ahead;                         // every warp walks the same requests and takes the same branches
        ahead = base + 32 + lane < a.n ? a.in[base + 32 + lane] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
        const uint32_t wp = mine.y & 0xFFu, wop = (mine.y >> 8) & 0xFFu;
        uint32_t live = __ballot_sync(0xFFFFFFFFu, wop == ISL_OP_ALLOC && wp < n_profiles && !((dead >> wp) & 1u));
        while (live) {
            const uint32_t j = __ffs(live) - 1;
            live &= live - 1;
            const uint32_t p = __shfl_sync(0xFFFFFFFFu, mine.y, j) & 0xFFu;
            if ((dead >> p) & 1u) continue;
            const uint32_t key = tree[(size_t)p * a.T + root];
            if (key == kInf) { dead |= 1u << p; continue; }
            const uint32_t v = key & 0xFFFFFFu;
            if (warp == 0) {                                 // the chain warp: the node's first GPU in range that admits p
                const uint32_t g0 = max(a.lo, __ldg(a.node_off + a.nlo + v)), g1 = min(a.hi, __ldg(a.node_off + a.nlo + v + 1));
                const uint32_t t = a.meta[v] >> 24;
                for (uint32_t gb = g0; gb < g1; gb += 32) {
                    const uint32_t g = gb + lane, o = g < g1 ? a.occ[g] : 0xFFu;
                    const uint32_t hit = __ballot_sync(0xFFFFFFFFu, g < g1 && admits(t, p, o));
                    if (!hit) continue;
                    if (lane == __ffs(hit) - 1) {
                        const uint32_t start = s_lut[(t * ISL_MAX_PROFILES + p) * 256 + o], size = s_sizes[t * ISL_MAX_PROFILES + p];
                        const uint32_t o2 = o | slice_span(start, size), wm = (1u << a.width[t]) - 1u;
                        a.occ[g] = (uint8_t)o2;
                        a.out[base + j] = pack_result(g, start, size, ISL_ST_PLACED);
                        a.busy[v] += __popc(o2 & wm) - __popc(o & wm);
                        s_ev[0] = o; s_ev[1] = o2;
                    }
                    ++placed;
                    break;
                }
            }
            __syncthreads();
            if (warp < n_profiles) {                          // warp q: profile q's fit count on the node, its leaf, its path to the root
                const uint32_t q = warp, o = s_ev[0], o2 = s_ev[1], meta = a.meta[v], t = meta >> 24;
                uint32_t* fq = a.fit + (size_t)q * a.Nr + v;
                const uint32_t f = *fq + admits(t, q, o2) - admits(t, q, o);
                uint32_t* tq = tree + (size_t)q * a.T;
                const uint32_t leaf = nodefit_leaf(f, a.busy[v], meta & 0xFFFFFFu, s_sizes[t * ISL_MAX_PROFILES + q], a.most, v);
                __syncwarp();
                if (lane == 0) { *fq = f; tq[v] = leaf; }
                uint32_t idx = v;
                for (uint32_t k = 0; k + 1 < a.levels; ++k) {
                    __syncwarp();
                    const uint32_t m = redux_min_u32(tq[a.lvl_off[k] + (idx & ~31u) + lane]);
                    idx >>= 5;
                    const uint32_t old = tq[a.lvl_off[k + 1] + idx];
                    if (old == m) break;                      // the ancestors keep their values
                    __syncwarp();
                    if (lane == 0) tq[a.lvl_off[k + 1] + idx] = m;
                }
            }
            __syncthreads();
        }
    }
    if (tid == 0) count_placed(a.ctrl, placed);
}

// ---------------------------------------------------------------------------------------------
// Gang topology: k_ganglocal (at the end of this file) and the per-gang bodies it runs (DESIGN.md 4.9-4.13).
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kGnThreads = 512;
constexpr uint32_t kGnMaxCtas = 160;                    // CTAs of one launch (at most one per SM)
constexpr unsigned long long kGnFail = 1ull << 63;
// A failed node's key in one- and few-node gangs: the deeper failure, then the lower node, is the smaller key
__device__ __forceinline__ unsigned long long gn_fail_key(uint32_t depth, uint32_t j) {
    return kGnFail | ((unsigned long long)(0x7FFFFFFFu - depth) << 32) | j;
}
__device__ __forceinline__ uint32_t gn_fail_depth(unsigned long long key) { return 0x7FFFFFFFu - (uint32_t)((key >> 32) & 0x7FFFFFFFu); }

struct GangNodeArgs {           // kernel parameter (by value)
    const uint2* in;            // requests (isl_request)
    uint2* out;                 // records: k_prepare's defaults, overwritten for the gang members
    uint8_t* occ;               // live occupancy (storage order)
    const uint8_t* gtab;        // table of every GPU's node (storage order)
    const uint8_t* lut;         // [table][profile][occ]: first legal start or ISL_START_NONE
    const uint8_t* score;       // [table][profile][occ]: what the policy minimises; zero for first-fit and right-to-left
    const uint8_t* sizes;       // [table][profile]
    const uint32_t* node_off;   // node offsets of the inventory in storage order
    const uint32_t* gang_off;   // n_gangs + 1
    uint8_t* scratch;           // Gr bytes: NodeShare::aux when the shares are in global memory
    unsigned long long* keys;   // [2][gridDim.x] per-CTA minima
    Ctrl* ctrl;
    uint32_t n_gangs, n_tables, lo, hi, nlo;   // the partition [lo, hi) in storage order, its first node
    uint32_t share;             // bytes of the largest share when the shares live in shared memory, 0 = global memory
    uint32_t cta_node[kGnMaxCtas + 1];
};

// k_ganglocal<.., kScore> on an ISL_FLAG_GANG_NODE_SCORE engine (DESIGN.md 4.16): what k_nodefit needs beside the gang arguments.  A
// struct of its own, so that the parameter block of every other k_ganglocal and of k_preempt_gangs keeps its layout; the host fills one
// for every launch, and the others read only its GangNodeArgs part, which comes first.
struct GangScoreArgs : GangNodeArgs {
    uint8_t width[kMaxTables];  // largest start + size over the rows of every table
    uint32_t most;              // 1: MostAllocated, 0: LeastAllocated
};

// Warp-wide: resolve the ALLOC members of requests [r0, r1) in order on the `cnt` bytes `b` of one node of table t, the engine's policy
// restricted to that node.  Returns how many leading ALLOC members were placed.  commit: b is the live share; the placements are also
// written to the occupancy (storage index gbase + position) and reported PLACED.
__device__ uint32_t gangnode_resolve(const GangNodeArgs& a, const DevProfiles& prof, uint8_t* b, uint32_t cnt, uint32_t gbase, uint32_t t,
                                     uint32_t r0, uint32_t r1, bool commit, uint32_t lane) {
    uint32_t depth = 0;
    for (uint32_t base = r0; base < r1; base += 32) {
        const uint2 q = base + lane < r1 ? a.in[base + lane] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
        uint32_t live = __ballot_sync(0xFFFFFFFFu, ((q.y >> 8) & 0xFFu) == ISL_OP_ALLOC);
        while (live) {
            const uint32_t j = __ffs(live) - 1;
            live &= live - 1;
            const uint32_t p = __shfl_sync(0xFFFFFFFFu, q.y, j) & 0xFFu;
            if (p >= prof.n) return depth;                  // an unknown profile fits nowhere
            const uint32_t row = (t * ISL_MAX_PROFILES + p) * 256;
            uint32_t key = kInf;
            for (uint32_t g = lane; g < cnt; g += 32) {
                const uint32_t o = b[g];
                if (__ldg(a.lut + row + o) != ISL_START_NONE) key = min(key, ((uint32_t)__ldg(a.score + row + o) << 24) | g);
            }
            const uint32_t m = redux_min_u32(key);         // every lane has read its bytes: the owner may rewrite one below
            if (m == kInf) return depth;
            const uint32_t g = m & 0xFFFFFFu;
            if ((g & 31u) == lane) {
                const uint32_t o = b[g], start = __ldg(a.lut + row + o), size = __ldg(a.sizes + t * ISL_MAX_PROFILES + p);
                const uint32_t o2 = o | slice_span(start, size);
                b[g] = (uint8_t)o2;
                if (commit) {
                    a.occ[gbase + g] = (uint8_t)o2;
                    a.out[base + j] = pack_result(flip_gpu(gbase + g, prof.flip), start, size, ISL_ST_PLACED);
                }
            }
            __syncwarp();
            ++depth;
        }
    }
    return depth;
}

// A CTA's share of the partition in k_ganglocal: the partition's nodes [j0, j1), which own its partition-local GPUs [base, base + cnt).
// `live` holds their committed bytes and `aux` a second byte per GPU (one- and few-node gangs: scratch copies, distinct-node gangs:
// node-used marks), both in shared memory, or in global memory when a share is too large for it (a.share == 0).  Every thread of the CTA
// builds it: the constructor copies the committed bytes into shared memory.
struct NodeShare {
    const GangNodeArgs& a;
    uint32_t j0, j1, base, cnt;
    uint8_t *live, *aux;
    __device__ __forceinline__ NodeShare(const GangNodeArgs& args, uint8_t* smem)
        : a(args), j0(args.cta_node[blockIdx.x]), j1(args.cta_node[blockIdx.x + 1]), base(nb(j0)), cnt(nb(j1) - base),
          live(args.share ? smem : args.occ + args.lo + base), aux(args.share ? smem + args.share : args.scratch + base) {
        if (a.share) for (uint32_t g = threadIdx.x; g < cnt; g += kGnThreads) live[g] = a.occ[a.lo + base + g];
    }
    // node j of the partition owns the partition-local GPUs [nb(j), nb(j + 1)); a node the partition cuts keeps its GPUs inside it
    __device__ __forceinline__ uint32_t nb(uint32_t j) const { return min(max(a.node_off[a.nlo + j], a.lo), a.hi) - a.lo; }
};

// Warp-wide (node-scored any-node and distinct-node members, DESIGN.md 4.16): node j's key for one member of profile p, nodefit_leaf over
// the node's busy slices under its table's width on the live bytes, with the partition-local position of the node's first GPU that
// admits p in place of the node.  One grid_min of these keys picks the highest score, then the lowest node, then that node's first
// admitting GPU: node-scoring rules 4-5.  kInf for an empty node, a node that admits nothing, and under `mark` a node marked `tag`.
__device__ __forceinline__ uint32_t gangscore_node(const GangScoreArgs& a, const NodeShare& sh, uint32_t j, uint32_t p, const uint8_t* mark,
                                                   uint32_t tag, uint32_t lane) {
    const uint32_t b0 = sh.nb(j) - sh.base, c = sh.nb(j + 1) - sh.base - b0;
    if (c == 0 || (mark && mark[b0] == tag)) return kInf;  // a used node's GPUs are all marked
    const uint32_t t = a.gtab[a.lo + sh.base + b0] & (kMaxTables - 1), row = (t * ISL_MAX_PROFILES + p) * 256;
    const uint32_t wm = (1u << a.width[t]) - 1u;
    uint32_t busy = 0, first = kInf;
    for (uint32_t g = lane; g < c; g += 32) {
        const uint32_t o = sh.live[b0 + g];
        busy += __popc(o & wm);
        if (__ldg(a.lut + row + o) != ISL_START_NONE) first = min(first, g);
    }
    busy = __reduce_add_sync(0xFFFFFFFFu, busy);
    first = redux_min_u32(first);
    return nodefit_leaf(first != kInf, busy, a.width[t] * c, __ldg(a.sizes + t * ISL_MAX_PROFILES + p), a.most, sh.base + b0 + first);
}

// Warp-wide, on a warp of the CTA that owns node j: commit the ALLOC members of requests [r, r1) on the node's live bytes (they stop by
// themselves where the evaluation on the scratch copy stopped).
__device__ __forceinline__ void gangnode_commit(const GangNodeArgs& a, const DevProfiles& prof, const NodeShare& sh, uint32_t j, uint32_t r,
                                                uint32_t r1, uint32_t lane) {
    const uint32_t b0 = sh.nb(j) - sh.base, c = sh.nb(j + 1) - sh.base - b0;
    gangnode_resolve(a, prof, sh.live + b0, c, a.lo + sh.base + b0, a.gtab[a.lo + sh.base + b0] & (kMaxTables - 1), r, r1, true, lane);
}

// One thread: request r, of profile p, takes its slices on the share's GPU g (partition-local sh.base + g) by the engine's policy: its
// live byte, the occupancy and a PLACED record.
__device__ __forceinline__ void commit_member(const GangNodeArgs& a, const DevProfiles& prof, const NodeShare& sh, uint32_t r, uint32_t p,
                                              uint32_t g) {
    const uint32_t t = a.gtab[a.lo + sh.base + g] & (kMaxTables - 1), row = (t * ISL_MAX_PROFILES + p) * 256, o = sh.live[g];
    const uint32_t start = __ldg(a.lut + row + o), size = __ldg(a.sizes + t * ISL_MAX_PROFILES + p);
    const uint32_t o2 = o | slice_span(start, size);
    sh.live[g] = (uint8_t)o2;
    a.occ[a.lo + sh.base + g] = (uint8_t)o2;
    a.out[r] = pack_result(flip_gpu(a.lo + sh.base + g, prof.flip), start, size, ISL_ST_PLACED);
}

// Warp-wide: a gang of requests [r0, r1) failed.  Every ALLOC member except the one of rank keep_rank among them is reported
// GANG_ABORTED; that one keeps k_prepare's NO_CAPACITY or BAD_PROFILE record.  kTrim (an elastic gang that commits its leading members,
// M3): only the ALLOC members of rank above keep_rank are written, and they report GANG_TRIMMED.
template <bool kTrim = false>
__device__ __forceinline__ void abort_gang_members(const uint2* in, uint2* out, const DevProfiles& prof, uint32_t r0, uint32_t r1,
                                                   uint32_t keep_rank, uint32_t lane) {
    uint32_t k = 0;                                         // ALLOC members before this block of 32
    for (uint32_t r = r0; r < r1; r += 32) {
        const uint32_t y = r + lane < r1 ? in[r + lane].y : (uint32_t)ISL_OP_NOOP << 8, p = y & 0xFFu;
        const bool alloc = ((y >> 8) & 0xFFu) == ISL_OP_ALLOC;
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, alloc), rank = k + __popc(ballot & ((1u << lane) - 1u));
        if (alloc && (kTrim ? rank > keep_rank : rank != keep_rank))
            out[r + lane] = pack_result(ISL_GPU_NONE, ISL_START_NONE, p < prof.n ? prof.rows[p].size : 0u, kTrim ? ISL_ST_GANG_TRIMMED : ISL_ST_GANG_ABORTED);
        k += __popc(ballot);
    }
}

// Warp-wide (few-node gangs): the request just past the d-th ALLOC member at or after request r (d >= 1, and [r, r1) holds that many).
__device__ __forceinline__ uint32_t skip_allocs(const uint2* in, uint32_t r, uint32_t r1, uint32_t d, uint32_t lane) {
    for (;; r += 32) {
        uint32_t ballot = __ballot_sync(0xFFFFFFFFu, r + lane < r1 && ((in[r + lane].y >> 8) & 0xFFu) == ISL_OP_ALLOC);
        const uint32_t c = __popc(ballot);
        if (d <= c) {
            for (; d > 1; --d) ballot &= ballot - 1;
            return r + __ffs(ballot);
        }
        d -= c;
    }
}
// Warp-wide (few-node and any-node gangs): a gang aborted after earlier rounds or members committed its ALLOC members among requests
// [r0, r1) as tentative PLACED records.  The CTA takes back those on its own nodes: the spans of one gang are disjoint and were free
// before it, so clearing them restores its live bytes and the occupancy, and it reports those members GANG_ABORTED (it is their records'
// only writer).  The records may come from other CTAs, written before a grid barrier of a later round, so they are read from L2.  One
// lane at a time writes, since two members may share a GPU.
__device__ void gangfew_undo(const GangNodeArgs& a, const NodeShare& sh, const DevProfiles& prof, uint32_t r0, uint32_t r1, uint32_t lane) {
    for (uint32_t r = r0; r < r1; r += 32) {
        const uint32_t i = r + lane;
        uint2 rec = make_uint2(ISL_GPU_NONE, (uint32_t)ISL_ST_GANG_ABORTED << 16);
        if (i < r1 && ((a.in[i].y >> 8) & 0xFFu) == ISL_OP_ALLOC) rec = __ldcg(a.out + i);
        const uint32_t pos = flip_gpu(rec.x, prof.flip) - a.lo - sh.base;     // inside this CTA's share when below sh.cnt
        uint32_t hits = __ballot_sync(0xFFFFFFFFu, (rec.y >> 16) == ISL_ST_PLACED && pos < sh.cnt);
        while (hits) {
            const uint32_t src = __ffs(hits) - 1;
            hits &= hits - 1;
            if (lane == src) {
                const uint32_t keep = ~slice_span(rec.y & 0xFFu, (rec.y >> 8) & 0xFFu), p = a.in[i].y & 0xFFu;
                sh.live[pos] &= (uint8_t)keep;
                a.occ[a.lo + sh.base + pos] &= (uint8_t)keep;
                a.out[i] = pack_result(ISL_GPU_NONE, ISL_START_NONE, prof.rows[p].size, ISL_ST_GANG_ABORTED);
            }
            __syncwarp();
        }
    }
}

// One gang of requests [r0, r1) of k_ganglocal of locality 1 (one node) or, kFew, 2 (few nodes), every thread of the CTA.  `scr`, the
// scratch copies, is the share's aux byte.  The shared words are the kernel's: s_warp and s_win for grid_min, s_need and s_allocs.
// One node (DESIGN.md 4.9): the gang commits on the first node, in the engine's scan order (storage order: ascending canonical,
// descending under ISL_POLICY_RIGHT_TO_LEFT), that takes all of its ALLOC members:
//   evaluate  one warp per node: copy the node's bytes to the scratch copy and count its free slices; a node with fewer free slices than
//             the gang's members need on its table is skipped (pass 0 only).  Otherwise the warp resolves the members in order on the
//             scratch copy, each one a warp min over the node's GPUs of score(t, p, o) << 24 | position (k_bestfit's lut and score tables; a
//             zero score table is first-fit).  Key: the node index for a success, else gn_fail_key(depth, node).
//   reduce    grid_min: the smallest key is the first node in scan order that takes the whole gang, or, with no such node, the deepest
//             failure.  When the winner of pass 0 is a failure every node is evaluated again without the filter (pass 1), since the
//             skipped nodes' depths are unknown.
//   commit    the warp 0 of the CTA that owns the winning node resolves the members again on the live bytes and writes the PLACED records
//             and the occupancy; a failure: CTA 0 reports every ALLOC member except the one at depth D GANG_ABORTED (that one keeps
//             k_prepare's NO_CAPACITY or BAD_PROFILE record).
// Few nodes (4.11): a loop of rounds over the gang's remaining members, from request ri on; each round is the evaluate and reduce steps
// above, and the winning key's depth d is how many members the round places (a success: all that remain).  The owner commits those d on
// its live bytes as tentative PLACED records and every CTA advances ri past d ALLOC members.  d = 0 aborts the gang without an undo log:
// each CTA takes back the tentative records on its own nodes (gangfew_undo), while CTA 0 reports the members after the one that found
// no node.
// kMin (k_ganglocal<kLocPerGang, true>, M3): a gang that fails at ALLOC member f >= min_m commits its first f members instead of aborting.
// One node: f is the deepest failure's depth D, and the owner of the first node that reaches it replays the members on its live bytes,
// which stop at D by themselves (the scratch copy started from the same bytes).  Few nodes: f is the members the earlier rounds placed.
// kScore (one node on an ISL_FLAG_GANG_NODE_SCORE engine, 4.16, N5): a node that takes the gang also counts its busy slices under its
// table's width (a second pass over its bytes), and its key is (100 - score(N, s_need[t])) << 32 | node, the gang scored as one pod;
// bit 63 stays clear, so every success still sorts before every failure.  Pass 0's filter stays valid: a node it skips cannot take the
// gang.
// kScore with kFew or kMin (ISL_FLAG_GANG_NODE_SCORE_ALL, 4.18, C4-C5): a failed node's key carries its score as well,
// kGnFail | (0x7FFFFFFF - d) << 32 | (100 - score(N, R_d)) << 24 | j, so the deepest nodes sort by score, then by node (j < 2^24: a
// node-scoring inventory has at most 2^20 nodes).  busy + R_d is the scratch copy's popcount under the width after the resolve, which
// gives the success key's score too.  That one key decides a few-node round and a one-node trim; one node without kMin keeps N5's keys.
template <bool kFew, bool kMin = false, bool kScore = false, class Args = GangNodeArgs>
__device__ __forceinline__ void gangnode_gang(const Args& a, const DevProfiles& prof, const NodeShare& sh, uint32_t r0, uint32_t r1,
                                              uint32_t& parity, uint32_t& placed, unsigned long long* s_warp, unsigned long long* s_win,
                                              uint32_t* s_need, uint32_t* s_allocs, uint32_t tid, uint32_t lane, uint32_t warp,
                                              uint32_t min_m = 0) {
    constexpr uint32_t kGnNodeMask = kScore ? 0xFFFFFFu : 0xFFFFFFFFu;    // the node in a failed key's low word
    uint8_t* const scr = sh.aux;
    uint32_t ri = r0, held = 0;     // kFew: the round's first request; members this CTA committed tentatively in earlier rounds
    uint32_t done = 0;              // kFew && kMin: members the earlier rounds placed (grid-uniform: the sum of the winning depths)
    for (;;) {                      // one round; without kFew every path leaves after the first
        if (tid < kMaxTables) s_need[tid] = 0;
        if (tid == 0) *s_allocs = 0;
        __syncthreads();                                    // also orders a commit of the previous gang or round before this one's reads
        uint32_t mine = 0;
        for (uint32_t r = ri + tid; r < r1; r += kGnThreads) {      // the slices the remaining ALLOCs take on a node of each table
            const uint32_t y = a.in[r].y, p = y & 0xFFu;
            if (((y >> 8) & 0xFFu) != ISL_OP_ALLOC) continue;
            ++mine;
            if (p < prof.n)
                for (uint32_t t = 0; t < a.n_tables; ++t) atomicAdd(&s_need[t], (uint32_t)__ldg(a.sizes + t * ISL_MAX_PROFILES + p));
        }
        if (mine) atomicAdd(s_allocs, mine);
        __syncthreads();
        const uint32_t allocs = *s_allocs;
        if (allocs == 0) break;                             // FREEs and NOOPs only: k_prepare's records stand
        unsigned long long win = ~0ull;
        for (uint32_t pass = 0; pass < 2; ++pass) {
            unsigned long long best = ~0ull;
            for (uint32_t j = sh.j0 + warp; j < sh.j1; j += kGnThreads / 32) {
                const uint32_t b0 = sh.nb(j) - sh.base, c = sh.nb(j + 1) - sh.base - b0;
                if (c == 0) continue;                       // an empty node places nothing: depth 0, the floor of every failure
                const uint32_t t = a.gtab[a.lo + sh.base + b0] & (kMaxTables - 1);
                uint32_t free_slices = 0;
                for (uint32_t g = lane; g < c; g += 32) {
                    const uint32_t o = sh.live[b0 + g];
                    scr[b0 + g] = (uint8_t)o;
                    free_slices += 8u - __popc(o);
                }
                free_slices = __reduce_add_sync(0xFFFFFFFFu, free_slices);
                if (pass == 0 && free_slices < s_need[t]) continue;
                const uint32_t d = gangnode_resolve(a, prof, scr + b0, c, a.lo + sh.base + b0, t, ri, r1, false, lane);
                if constexpr (kScore && (kFew || kMin)) {   // busy + R_d: the scratch copy's slices under the width after the d members
                    uint32_t busy = 0;
                    for (uint32_t g = lane; g < c; g += 32) busy += __popc(scr[b0 + g] & ((1u << a.width[t]) - 1u));
                    busy = __reduce_add_sync(0xFFFFFFFFu, busy);
                    const unsigned long long score = nodefit_leaf(1u, busy, a.width[t] * c, 0u, a.most, 0u) >> 24;     // 100 - score
                    best = min(best, d == allocs ? score << 32 | j : gn_fail_key(d, 0u) | score << 24 | j);
                } else if constexpr (kScore) {     // the node's busy slices under its width on the live bytes, before the gang
                    uint32_t busy = 0;
                    for (uint32_t g = lane; g < c; g += 32) busy += __popc(sh.live[b0 + g] & ((1u << a.width[t]) - 1u));
                    busy = __reduce_add_sync(0xFFFFFFFFu, busy);
                    const unsigned long long score = nodefit_leaf(1u, busy, a.width[t] * c, s_need[t], a.most, 0u) >> 24;     // 100 - score
                    best = min(best, d == allocs ? score << 32 | j : gn_fail_key(d, j));
                } else {
                    best = min(best, d == allocs ? (unsigned long long)j : gn_fail_key(d, j));
                }
            }
            win = grid_min<kGnThreads>(best, a.keys, parity, s_warp, s_win);
            if (!(win & kGnFail)) break;                    // a node takes the whole gang: the skipped nodes could not have come first
        }
        if (!(win & kGnFail)) {
            const uint32_t j = (uint32_t)win;
            if (j >= sh.j0 && j < sh.j1 && warp == 0) {     // the owner commits on its live bytes
                gangnode_commit(a, prof, sh, j, ri, r1, lane);
                placed += allocs;
            }
            if (kFew) placed += held;                       // the gang commits: its tentative members count
            break;
        }
        if constexpr (!kFew) {
            if constexpr (kMin) {
                const uint32_t d = gn_fail_depth(win), j = (uint32_t)win & kGnNodeMask;
                if (d >= min_m) {                           // min_m >= 1, so ~0ull (depth 0) never gets here
                    if (j >= sh.j0 && j < sh.j1 && warp == 0) {
                        gangnode_commit(a, prof, sh, j, ri, r1, lane);
                        placed += d;
                    }
                    if (blockIdx.x == 0 && warp == 0) abort_gang_members<true>(a.in, a.out, prof, r0, r1, d, lane);
                    break;
                }
            }
            if (blockIdx.x == 0 && warp == 0)               // the deepest failure's depth; ~0ull (no node evaluated) is depth 0 as well
                abort_gang_members(a.in, a.out, prof, r0, r1, gn_fail_depth(win), lane);
            break;
        } else {
            const uint32_t d = gn_fail_depth(win), j = (uint32_t)win & kGnNodeMask;      // members the round places
            if (kMin && d == 0 && done >= min_m) {          // the earlier rounds' members commit, m_i keeps its record
                placed += held;
                if (blockIdx.x == 0 && warp == 0) abort_gang_members<true>(a.in, a.out, prof, ri, r1, 0, lane);
                break;
            }
            if (d == 0) {                                   // no node takes m_i: every CTA takes back its tentative members
                if (warp == 0) gangfew_undo(a, sh, prof, r0, ri, lane);
                if (blockIdx.x == 0 && warp == 0) abort_gang_members(a.in, a.out, prof, ri, r1, 0, lane);
                break;
            }
            if (j >= sh.j0 && j < sh.j1 && warp == 0) {     // the owner commits the round's d members on its live bytes
                gangnode_commit(a, prof, sh, j, ri, r1, lane);
                held += d;
            }
            ri = skip_allocs(a.in, ri, r1, d, lane);        // every CTA read the same key: all advance alike
            done += d;
        }
    }
}

// One gang of requests [r0, r1) of k_ganglocal of locality 3 (distinct nodes, DESIGN.md 4.10), every thread of the CTA: the ALLOC
// members are resolved in order, each by the engine's policy restricted to the partition's GPUs whose node holds no earlier member of
// the same gang.  So no member ever sees another member's slices: a member's key on a GPU depends only on the committed bytes, and the
// gang needs no scratch copy and no rollback.  Per ALLOC member:
//   choose    every CTA takes the minimum of score(t, p, o) << 24 | partition-local storage position over its GPUs not marked used
//             (k_bestfit's lut and score tables; a zero score table is first-fit, and right-to-left is the ascending scan of its reversed
//             storage); grid_min over the CTAs' 32-bit minima gives every CTA the member's GPU.
//   mark      the CTA that owns that GPU marks its node's GPUs with the gang's tag and pushes (request, GPU) onto its stack of wins.
// A member with no GPU ends the gang: it keeps k_prepare's record (NO_CAPACITY or BAD_PROFILE), CTA 0 reports every other ALLOC member
// GANG_ABORTED, and no occupancy byte is written.  Otherwise every CTA writes the bytes and PLACED records of its stack.
// `tag` (1..255) marks the nodes the gang uses in the share's aux byte; tag 1 clears the marks first, so a mark can only equal `tag` when
// this gang wrote it.  `dead`: profiles no GPU of the partition admits any more.  The shared words are the kernel's: s_warp and s_win for
// grid_min, and the size of the CTA's stack of wins, which is 0 between gangs.  kMin (k_ganglocal<kLocPerGang, true>, M3): a member that
// finds no GPU at rank fail >= min_m commits the stack of wins, which holds the members before it, as a success does.
// kScore (ISL_FLAG_GANG_NODE_SCORE, 4.16, N4): choose takes gangscore_node's key, one warp per unmarked node of the share.
template <bool kMin = false, bool kScore = false, class Args = GangNodeArgs>
__device__ __forceinline__ void gangspread_gang(const Args& a, const DevProfiles& prof, const NodeShare& sh, uint2* wins, uint32_t r0,
                                                uint32_t r1, uint32_t tag, uint32_t& parity, uint32_t& placed, uint32_t& dead,
                                                uint32_t* s_warp, uint32_t* s_win, uint32_t* s_nwins, uint32_t tid, uint32_t lane,
                                                uint32_t warp, uint32_t min_m = 0) {
    const uint32_t base = sh.base, cnt = sh.cnt;
    uint8_t* const mark = sh.aux;                           // tag of the gang whose member uses the GPU's node
    if (tag == 1u) for (uint32_t g = tid; g < cnt; g += kGnThreads) mark[g] = 0;
    __syncthreads();                                        // also orders the previous gang's commit before this gang's reads
    uint32_t rank = 0, fail = kInf;                         // ALLOC members resolved so far; the rank of the one that found no GPU
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t y = a.in[r].y, p = y & 0xFFu;
        if (((y >> 8) & 0xFFu) != ISL_OP_ALLOC) continue;
        uint32_t win = kInf;                                // an unknown or dead profile fails without a barrier: every CTA knows it
        if (p < prof.n && !((dead >> p) & 1u)) {
            uint32_t key = kInf;
            if constexpr (kScore) {
                for (uint32_t j = sh.j0 + warp; j < sh.j1; j += kGnThreads / 32) key = min(key, gangscore_node(a, sh, j, p, mark, tag, lane));
            } else {
                for (uint32_t g = tid; g < cnt; g += kGnThreads) {
                    if (mark[g] == tag) continue;
                    const uint32_t o = sh.live[g], t = a.n_tables > 1 ? a.gtab[a.lo + base + g] & (kMaxTables - 1) : 0u;
                    const uint32_t row = (t * ISL_MAX_PROFILES + p) * 256;
                    if (__ldg(a.lut + row + o) != ISL_START_NONE) key = min(key, ((uint32_t)__ldg(a.score + row + o) << 24) | (base + g));
                }
            }
            win = grid_min<kGnThreads>(key, a.keys, parity, s_warp, s_win);
            if (win == kInf && rank == 0) dead |= 1u << p;
        }
        if (win == kInf) { fail = rank; break; }
        const uint32_t pos = (win & 0xFFFFFFu) - base;
        if (pos < cnt) {                                    // this CTA owns the member's node: the node is used for the rest of the gang
            uint32_t jl = sh.j0, jh = sh.j1;                // nb(jl) <= base + pos < nb(jh): the last such jl is the non-empty node
            while (jh - jl > 1) {
                const uint32_t mid = (jl + jh) / 2;
                if (sh.nb(mid) - base <= pos) jl = mid; else jh = mid;
            }
            for (uint32_t g = sh.nb(jl) - base + tid; g < sh.nb(jl + 1) - base; g += kGnThreads) mark[g] = (uint8_t)tag;
            if (tid == 0) wins[sh.j0 + (*s_nwins)++] = make_uint2(r, pos);     // one win per node of the CTA: the stack fits its nodes
        }
        __syncthreads();                                    // the marks and the stack are in place before the next member's scan
        ++rank;
    }
    const bool trim = kMin && fail != kInf && fail >= min_m;
    if (fail == kInf || trim) {                             // commit: each CTA writes its members; their nodes, hence GPUs, differ
        const uint32_t nw = *s_nwins;
        for (uint32_t k = tid; k < nw; k += kGnThreads) {
            const uint2 w = wins[sh.j0 + k];
            commit_member(a, prof, sh, w.x, a.in[w.x].y & 0xFFu, w.y);
        }
        placed += nw;
        if (trim && blockIdx.x == 0 && warp == 0) abort_gang_members<true>(a.in, a.out, prof, r0, r1, fail, lane);
    } else if (blockIdx.x == 0 && warp == 0) {              // the member at rank `fail` keeps its record, every other ALLOC member aborts
        abort_gang_members(a.in, a.out, prof, r0, r1, fail, lane);
    }
    __syncthreads();                                        // every thread has read the stack's size
    if (tid == 0) *s_nwins = 0;
}

// One gang of locality 0: every CTA takes the minimum of score(t, p, o) << 24 | partition-local storage position over its live bytes
// (locality 3's key with no GPU masked), grid_min gives every CTA the member's GPU, and the CTA that owns it commits the member
// tentatively to its live share, the occupancy and a PLACED record.  A member with no GPU aborts the gang: every CTA takes back the
// tentative members on its own nodes (gangfew_undo), and CTA 0 reports the members after the failing one GANG_ABORTED.  An unknown or
// dead profile fails without a barrier: gangfew_undo only touches records on the CTA's own nodes, which that CTA wrote itself.
// kMin (k_ganglocal<kLocPerGang, true>, M3): a member with no GPU at rank >= min_m keeps the tentative members, which then commit.
// kScore (ISL_FLAG_GANG_NODE_SCORE, 4.16, N3): the key is gangscore_node's, one warp per node of the share, on the live bytes, so each
// member sees the gang's tentative members in its nodes' busy slices.  No per-node state outlives a member, so gangfew_undo is unchanged.
template <bool kMin = false, bool kScore = false, class Args = GangNodeArgs>
__device__ __forceinline__ void ganglocal_any(const Args& a, const DevProfiles& prof, const NodeShare& sh, uint32_t r0, uint32_t r1,
                                              uint32_t& parity, uint32_t& placed, uint32_t& dead, uint32_t* s_warp, uint32_t* s_win,
                                              uint32_t tid, uint32_t lane, uint32_t warp, uint32_t min_m = 0) {
    const uint32_t base = sh.base, cnt = sh.cnt;
    __syncthreads();                                        // the previous gang's commits are in the live share before this gang's reads
    uint32_t rank = 0;                                      // ALLOC members committed tentatively so far
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t y = a.in[r].y, p = y & 0xFFu;
        if (((y >> 8) & 0xFFu) != ISL_OP_ALLOC) continue;
        uint32_t win = kInf;
        if (p < prof.n && !((dead >> p) & 1u)) {
            uint32_t key = kInf;
            if constexpr (kScore) {
                for (uint32_t j = sh.j0 + warp; j < sh.j1; j += kGnThreads / 32) key = min(key, gangscore_node(a, sh, j, p, nullptr, 0u, lane));
            } else {
                for (uint32_t g = tid; g < cnt; g += kGnThreads) {
                    const uint32_t o = sh.live[g], t = a.n_tables > 1 ? a.gtab[a.lo + base + g] & (kMaxTables - 1) : 0u;
                    const uint32_t row = (t * ISL_MAX_PROFILES + p) * 256;
                    if (__ldg(a.lut + row + o) != ISL_START_NONE) key = min(key, ((uint32_t)__ldg(a.score + row + o) << 24) | (base + g));
                }
            }
            win = grid_min<kGnThreads>(key, a.keys, parity, s_warp, s_win);
            if (win == kInf && rank == 0) dead |= 1u << p;  // no tentative slice of this gang is in the way
        }
        if (win == kInf) {
            if (kMin && rank >= min_m) {
                if (blockIdx.x == 0) {
                    placed += rank;
                    if (warp == 0) abort_gang_members<true>(a.in, a.out, prof, r, r1, 0, lane);
                }
                return;
            }
            if (warp == 0) gangfew_undo(a, sh, prof, r0, r, lane);
            if (blockIdx.x == 0 && warp == 0) abort_gang_members(a.in, a.out, prof, r, r1, 0, lane);
            return;
        }
        const uint32_t pos = (win & 0xFFFFFFu) - base;
        if (pos < cnt && tid == 0) commit_member(a, prof, sh, r, p, pos);     // the owner commits the member tentatively
        __syncthreads();                                    // the commit is in the live share before the next member's scan
        ++rank;
    }
    if (blockIdx.x == 0) placed += rank;                    // the gang commits: CTA 0 counts its members once
}

// Balanced gangs (ISL_FLAG_GANG_BALANCED, DESIGN.md 4.17): node j of the partition holds wins[j] = (count, tag), the number of ALLOC
// members of the running gang placed on it, valid only when `tag` is that gang's kBalTag | gang index.  k_ganglocal<.., kBal> clears the
// words of its nodes once per launch; a distinct-node stack writes a share position, below 2^24, into the second word.  So no count
// outlives its gang, and none is ever reset.
constexpr uint32_t kBalTag = 1u << 31;
__device__ __forceinline__ uint32_t gangbalance_count(const uint2* wins, uint32_t j, uint32_t tag) {
    const uint2 w = wins[j];
    return w.y == tag ? w.x : 0u;
}

// Warp-wide over the nodes of the share this warp visits, over the GPUs that admit p: with lim == kInf the least count << 32 | key, else
// the least key alone over the nodes whose count is at most lim, where key is ganglocal_any's score << 24 | partition-local storage
// position; ~0ull when there is none.  (A lane visits many nodes: with the count above a filtered key, its minimum would be the key of
// its least-count node, not its least key.)  kScore (ISL_FLAG_GANG_NODE_SCORE_ALL, 4.18, C6): the key below the count is gangscore_node's,
// so the nodes within the skew sort by score, then node, and the member takes its node's first admitting GPU.
template <bool kScore = false, class Args = GangNodeArgs>
__device__ __forceinline__ unsigned long long gangbalance_key(const Args& a, const NodeShare& sh, const uint2* wins, uint32_t p, uint32_t tag,
                                                             uint32_t lim, uint32_t lane, uint32_t warp) {
    unsigned long long key = ~0ull;
    for (uint32_t j = sh.j0 + warp; j < sh.j1; j += kGnThreads / 32) {
        const uint32_t b0 = sh.nb(j) - sh.base, c = sh.nb(j + 1) - sh.base - b0;
        if (c == 0) continue;
        const uint32_t n = gangbalance_count(wins, j, tag);
        if (n > lim) continue;
        const unsigned long long hi = lim == kInf ? (unsigned long long)n << 32 : 0ull;
        if constexpr (kScore) {
            const uint32_t s = gangscore_node(a, sh, j, p, nullptr, 0u, lane);
            if (s != kInf) key = min(key, hi | s);
            continue;
        }
        const uint32_t t = a.n_tables > 1 ? a.gtab[a.lo + sh.base + b0] & (kMaxTables - 1) : 0u, row = (t * ISL_MAX_PROFILES + p) * 256;
        for (uint32_t g = lane; g < c; g += 32) {
            const uint32_t o = sh.live[b0 + g];
            if (__ldg(a.lut + row + o) != ISL_START_NONE)
                key = min(key, hi | ((uint32_t)__ldg(a.score + row + o) << 24) | (sh.base + b0 + g));
        }
    }
    return key;
}

// One gang of a balanced locality byte (4..255, maxSkew skew = byte - 3; B2): ganglocal_any's member-by-member tentative commits, each
// member restricted to the nodes whose count is at most mu + skew - 1, mu the least count over the nodes that admit it.  Per member:
//   skew 1    one 64-bit grid_min of gangbalance_key: the least count first, then ganglocal_any's key among the nodes that have it;
//   skew > 1  a 32-bit grid_min of the counts in those keys gives mu, a second one the least key over the nodes at most mu + skew - 1.
// The CTA that owns the winning GPU commits the member (commit_member) and adds one to its node's count.  A node at mu always takes part,
// so a member finds no GPU only where none admits it: the failure, the dead-profile mask and kMin's trim (B5) are ganglocal_any's.
// kScore (C6): the keys are gangbalance_key<true>'s, the node score among the nodes within the skew.
template <bool kMin = false, bool kScore = false, class Args = GangNodeArgs>
__device__ __forceinline__ void gangbalance_gang(const Args& a, const DevProfiles& prof, const NodeShare& sh, uint2* wins, uint32_t r0,
                                                 uint32_t r1, uint32_t tag, uint32_t skew, uint32_t& parity, uint32_t& placed, uint32_t& dead,
                                                 unsigned long long* s_warp64, unsigned long long* s_win64, uint32_t* s_warp32,
                                                 uint32_t* s_win32, uint32_t tid, uint32_t lane, uint32_t warp, uint32_t min_m = 0) {
    const uint32_t base = sh.base, cnt = sh.cnt;
    __syncthreads();                                        // the previous gang's commits are in the live share before this gang's reads
    uint32_t rank = 0;                                      // ALLOC members committed tentatively so far
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t y = a.in[r].y, p = y & 0xFFu;
        if (((y >> 8) & 0xFFu) != ISL_OP_ALLOC) continue;
        uint32_t win = kInf;
        if (p < prof.n && !((dead >> p) & 1u)) {
            if (skew == 1) {
                const unsigned long long w = grid_min<kGnThreads>(gangbalance_key<kScore>(a, sh, wins, p, tag, kInf, lane, warp), a.keys,
                                                                  parity, s_warp64, s_win64);
                win = (uint32_t)w;                          // kInf when no GPU admits p
            } else {
                const uint32_t mu = grid_min<kGnThreads>((uint32_t)(gangbalance_key<kScore>(a, sh, wins, p, tag, kInf, lane, warp) >> 32),
                                                         a.keys, parity, s_warp32, s_win32);
                if (mu != kInf)
                    win = grid_min<kGnThreads>((uint32_t)gangbalance_key<kScore>(a, sh, wins, p, tag, mu + skew - 1u, lane, warp), a.keys,
                                               parity, s_warp32, s_win32);
            }
            if (win == kInf && rank == 0) dead |= 1u << p;  // no tentative slice of this gang is in the way
        }
        if (win == kInf) {
            if (kMin && rank >= min_m) {
                if (blockIdx.x == 0) {
                    placed += rank;
                    if (warp == 0) abort_gang_members<true>(a.in, a.out, prof, r, r1, 0, lane);
                }
                return;
            }
            if (warp == 0) gangfew_undo(a, sh, prof, r0, r, lane);
            if (blockIdx.x == 0 && warp == 0) abort_gang_members(a.in, a.out, prof, r, r1, 0, lane);
            return;
        }
        const uint32_t pos = (win & 0xFFFFFFu) - base;
        if (pos < cnt && tid == 0) {                        // the owner commits the member tentatively and counts it on its node
            commit_member(a, prof, sh, r, p, pos);
            uint32_t jl = sh.j0, jh = sh.j1;                // nb(jl) <= base + pos < nb(jh): the last such jl is the non-empty node
            while (jh - jl > 1) {
                const uint32_t mid = (jl + jh) / 2;
                if (sh.nb(mid) - base <= pos) jl = mid; else jh = mid;
            }
            wins[jl] = make_uint2(gangbalance_count(wins, jl, tag) + 1u, tag);
        }
        __syncthreads();                                    // the commit and the count are in place before the next member's scan
        ++rank;
    }
    if (blockIdx.x == 0) placed += rank;                    // the gang commits: CTA 0 counts its members once
}

// ---------------------------------------------------------------------------------------------
// k_ganglocal: isl_place_gangs on an engine created with a gang-topology flag (DESIGN.md 4.9-4.13).  One cooperative launch per call
// behind k_prepare (frees and default records).  CTA c owns the partition's nodes [cta_node[c], cta_node[c + 1]) (whole nodes, balanced
// by GPU count on the host) and keeps their occupancy bytes and a second byte per GPU in shared memory, or in global memory when a share
// is too large for it (NodeShare).  The gangs run in array order, each on the occupancy the earlier ones left.  kLoc is every gang's
// locality, or kLocPerGang for each gang's own byte:
//   ISL_GANG_ONE_NODE        gangnode_gang<false>   ISL_FLAG_GANG_ONE_NODE (4.9): every member on one node
//   ISL_GANG_FEW_NODES       gangnode_gang<true>    ISL_FLAG_GANG_FEW_NODES (4.11): one node when one takes the gang, else few nodes
//   ISL_GANG_DISTINCT_NODES  gangspread_gang        ISL_FLAG_GANG_DISTINCT_NODES (4.10): every member on a different node
//   kLocPerGang              locality[gi]           ISL_FLAG_GANG_LOCALITY (4.12): the byte of gang gi (checked on the host) is 1, 2 or 3
//                                                   as above or 0, ganglocal_any: rules 2-4, member by member over the whole share
// kMin (kLocPerGang only): every call on an ISL_FLAG_GANG_MIN_MEMBERS engine (4.13), whatever its locality flag.  The host writes the
// engine's locality into every gang's byte (or the gang's own under ISL_FLAG_GANG_LOCALITY), and each gang's effective minimum m' (M1)
// as a uint32 right after the bytes, rounded up to 4; a gang that fails at ALLOC member f >= m' commits its first f members (M3).
// With a constant kLoc the compiler drops the other branches and their shared words.
// Every barrier depends only on the gang offsets, the locality bytes, the minima and the winning keys, which every CTA reads alike, so
// every branch is grid-uniform.  The scratch copies of localities 1 and 2 overwrite the aux bytes, so the distinct-node tags count
// locality-3 gangs and restart at 1, which clears the marks, after every locality-1 or -2 gang, whose scratch copies may equal any tag;
// on their own the tags run 1..255 and the marks are cleared once every 255 gangs.  The dead-profile mask is shared by localities 0 and
// 3: a bit is set only when a gang's first ALLOC member finds no GPU, on a state without tentative slices; after k_prepare's FREEs the
// occupancy only grows and an abort restores it exactly, so the bit stays valid.  Every record has one writer: the CTA that owns a GPU
// writes the PLACED records on it and rewrites its own tentative ones GANG_ABORTED when the gang aborts (gangfew_undo); CTA 0 writes
// GANG_ABORTED or GANG_TRIMMED for the other members, except the one that stopped the gang, which keeps k_prepare's NO_CAPACITY or
// BAD_PROFILE record.
// kScore (an ISL_FLAG_GANG_NODE_SCORE engine, 4.16): the bodies put the node score in their keys, and `a` carries the widths and the
// policy (GangScoreArgs).  Without ISL_FLAG_GANG_NODE_SCORE_ALL (kLoc ISL_GANG_ANY_NODES, _ONE_NODE, _DISTINCT_NODES or kLocPerGang,
// never with kMin) the host refuses a few-node byte, so the few-node branch is never taken; with it (4.18) kLoc may also be
// ISL_GANG_FEW_NODES, and kMin and kBal may come with kScore.
// kBal (kLocPerGang on an ISL_FLAG_GANG_BALANCED engine, 4.17, with or without kMin): a byte of 4..255 is a balanced gang,
// gangbalance_gang with maxSkew byte - 3; its per-node counts are in `wins`, whose words of the CTA's nodes it clears first.  It leaves
// the aux bytes alone, so the distinct-node tags run on across it.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kLocPerGang = 4;
template <uint32_t kLoc, bool kMin = false, bool kScore = false, bool kBal = false>
__global__ void __launch_bounds__(kGnThreads, 1) k_ganglocal(std::conditional_t<kScore, GangScoreArgs, GangNodeArgs> a, DevProfiles prof, uint2* wins,
                                                             const uint8_t* __restrict__ locality) {
    static_assert(!kBal || kLoc == kLocPerGang, "balanced gangs are per-gang bytes");
    extern __shared__ __align__(16) uint8_t gl_smem[];
    __shared__ unsigned long long s_warp64[kGnThreads / 32];
    __shared__ unsigned long long s_win64;
    __shared__ uint32_t s_warp32[kGnThreads / 32];
    __shared__ uint32_t s_win32, s_nwins, s_need[kMaxTables], s_allocs;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const NodeShare sh(a, gl_smem);
    if (tid == 0) s_nwins = 0;
    if constexpr (kBal) for (uint32_t j = sh.j0 + tid; j < sh.j1; j += kGnThreads) wins[j] = make_uint2(0u, 0u);
    uint32_t parity = 0, placed = 0, dead = 0, spread = 0;  // spread: locality-3 gangs since the marks were last cleared
    for (uint32_t gi = 0; gi < a.n_gangs; ++gi) {
        const uint32_t r0 = __ldg(a.gang_off + gi), r1 = __ldg(a.gang_off + gi + 1), loc = kLoc == kLocPerGang ? __ldg(locality + gi) : kLoc;
        const uint32_t min_m = kMin ? __ldg(reinterpret_cast<const uint32_t*>(locality + ((a.n_gangs + 3u) & ~3u)) + gi) : 0u;
        if (loc == ISL_GANG_ONE_NODE || loc == ISL_GANG_FEW_NODES) {
            if (loc == ISL_GANG_ONE_NODE)
                gangnode_gang<false, kMin, kScore>(a, prof, sh, r0, r1, parity, placed, s_warp64, &s_win64, s_need, &s_allocs, tid, lane, warp,
                                                   min_m);
            else gangnode_gang<true, kMin, kScore>(a, prof, sh, r0, r1, parity, placed, s_warp64, &s_win64, s_need, &s_allocs, tid, lane, warp,
                                                   min_m);
            spread = 0;                                     // the scratch copies overwrote the marks
        } else if (loc == ISL_GANG_DISTINCT_NODES) {
            gangspread_gang<kMin, kScore>(a, prof, sh, wins, r0, r1, 1u + spread % 255u, parity, placed, dead, s_warp32, &s_win32, &s_nwins, tid,
                                          lane, warp, min_m);
            ++spread;
        } else if (kBal && loc > ISL_GANG_DISTINCT_NODES) {
            gangbalance_gang<kMin, kScore>(a, prof, sh, wins, r0, r1, kBalTag | gi, loc - ISL_GANG_DISTINCT_NODES, parity, placed, dead,
                                           s_warp64, &s_win64, s_warp32, &s_win32, tid, lane, warp, min_m);
        } else {
            ganglocal_any<kMin, kScore>(a, prof, sh, r0, r1, parity, placed, dead, s_warp32, &s_win32, tid, lane, warp, min_m);
        }
    }
    if (tid == 0 && placed) count_placed(a.ctrl, placed);
}

// ---------------------------------------------------------------------------------------------
// Gang preemption: isl_preempt on an ISL_FLAG_GANG_PREEMPT engine (DESIGN.md 4.15), after k_victim_map.  One cooperative launch per call
// on k_ganglocal's node-aligned shares: CTA c owns the partition's nodes [cta_node[c], cta_node[c + 1]) (NodeShare; only its node bounds
// are used, since a query writes no occupancy byte).  Each GPU of a share keeps k_preempt's 11 bytes (priority of every slice's victim,
// 255 = none; occupancy; run starts; table) and a scratch copy of the first 10, in shared memory when the share fits the opt-in, else in
// global memory (kPgBytesPerGpu per GPU of the partition).  The gangs run in array order, each on the state the committed ones left:
//   any node / distinct nodes  pg_members: per ALLOC member one grid_min of preempt_key over the share; the owner of the winning GPU logs
//                              its prior state (one PgLog per member), applies the eviction and writes the record and evict row.
//                              Distinct nodes also mark the winning node as used for the rest of the gang (in the scratch occupancy
//                              byte).  A member with no candidate rolls the gang back from the log in reverse order.
//   one node                   pg_one_node: one warp per node resolves the members on the scratch copy of its node, accumulating the
//                              cost (max, sum, count of the victims); a two-word grid_min picks the node; its owner replays the gang on
//                              its live state.
// Records: every CTA writes the defaults of its slice of the requests (NOOP, BAD_PROFILE, NO_CAPACITY) before one grid barrier; the
// host has set every evict row to ISL_GPU_NONE.  A PLACED record and its row have one writer, the CTA that owns the GPU; CTA 0 writes
// GANG_ABORTED for the members after the one that stopped a gang.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kPgBytesPerGpu = 21;                 // 11 live bytes + 10 scratch bytes per GPU of a share

struct PgLog {                  // a GPU's state before an any-node or distinct-node member took it (the rollback log, one per member)
    unsigned long long prio;
    uint32_t r, gw, o_rs, pad;  // the member's request, the partition-local GPU, occupancy | run starts << 8
};

struct PgState {                // one copy of the per-GPU state of a share, indexed by share position
    unsigned long long* prio;
    uint8_t *occ, *rs;
};

// The best candidate of one GPU for a preemptor of profile p at priority pi (k_preempt's scan of one GPU): ~0 when there is none.
__device__ __forceinline__ unsigned long long pg_best(const uint8_t* s_masks, uint32_t tab, uint32_t p, uint32_t pi, unsigned long long pr,
                                                      uint32_t o, uint32_t rs, uint32_t gw) {
    uint32_t ev = 0;                                        // slices whose victim has a priority below the preemptor's
#pragma unroll
    for (uint32_t s = 0; s < ISL_SLOTS; ++s) ev |= (((uint32_t)(pr >> (8 * s)) & 0xFFu) < pi) << s;
    const uint32_t blocked = o & ~ev;
    const uint8_t* mk = s_masks + (tab * ISL_MAX_PROFILES + p) * ISL_MAX_STARTS;
    unsigned long long best = ~0ull;
#pragma unroll
    for (uint32_t k = 0; k < ISL_MAX_STARTS; ++k) {
        const uint32_t m = mk[k];
        if (m && !(m & blocked)) best = min(best, preempt_key(m, o, rs, pr, gw, k));
    }
    return best;
}

// One thread: the preemptor of request r takes span m on share position g (partition-local GPU gw) of state st: its victims leave whole,
// the span becomes busy and pinned.  rec: also write the PLACED record and the evict row (victim indices ascending).
__device__ __forceinline__ void pg_take(const PreemptArgs& p, const DevProfiles& prof, const PgState& st, uint32_t g, uint32_t gw, uint32_t m,
                                        uint32_t r, bool rec) {
    const uint32_t o = st.occ[g], rs = st.rs[g];
    const uint32_t heads = (rs & m) | (o & m & (m & (0u - m)));
    const uint4* w4 = reinterpret_cast<const uint4*>(p.vmap + (size_t)gw * ISL_SLOTS);
    const uint4 w0 = w4[0], w1 = w4[1];
    const uint32_t w[ISL_SLOTS] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
    uint32_t idx[ISL_SLOTS], nv = 0, gone = 0;
    for (uint32_t h = heads; h; h &= h - 1) {
        const uint32_t v = w[__ffs(h) - 1];
        uint32_t j = nv++;
        for (; j > 0 && idx[j - 1] > v; --j) idx[j] = idx[j - 1];
        idx[j] = v;
#pragma unroll
        for (uint32_t s = 0; s < ISL_SLOTS; ++s) gone |= (w[s] == v) << s;
    }
    const uint32_t touched = gone | m;
    unsigned long long pr = st.prio[g];
#pragma unroll
    for (uint32_t s = 0; s < ISL_SLOTS; ++s) if ((touched >> s) & 1u) pr |= 0xFFull << (8 * s);
    st.prio[g] = pr; st.rs[g] = (uint8_t)(rs & ~touched); st.occ[g] = (uint8_t)((o & ~gone) | m);
    if (rec) {
        p.out[r] = pack_result(flip_gpu(p.lo + gw, prof.flip), __ffs(m) - 1, __popc(m), ISL_ST_PLACED);
        for (uint32_t j = 0; j < nv; ++j) p.evict[(size_t)r * ISL_SLOTS + j] = idx[j];
    }
}

// Warp-wide: resolve the ALLOC members of requests [r0, r1) in order by rules 4-5 restricted to the c GPUs at share positions [b0, b0 + c)
// of state st (one node).  Returns how many leading ALLOC members got a candidate; *all: every one did.  mx, sum, cnt: the highest
// victim priority + 1, the sum of the priorities and the number of the victims they evict.  commit: also write records and evict rows.
__device__ uint32_t pg_node_resolve(const PreemptArgs& p, const DevProfiles& prof, const PgState& st, const uint8_t* tab, const uint8_t* s_masks,
                                    uint32_t b0, uint32_t c, uint32_t base, uint32_t r0, uint32_t r1, bool commit, uint32_t lane, bool* all,
                                    uint32_t& mx, uint32_t& sum, uint32_t& cnt) {
    uint32_t depth = 0;
    mx = sum = cnt = 0;
    *all = false;
    for (uint32_t rb = r0; rb < r1; rb += 32) {
        const uint2 q = rb + lane < r1 ? p.in[rb + lane] : make_uint2(0, (uint32_t)ISL_OP_NOOP << 8);
        uint32_t live = __ballot_sync(0xFFFFFFFFu, ((q.y >> 8) & 0xFFu) == ISL_OP_ALLOC);
        while (live) {
            const uint32_t j = __ffs(live) - 1;
            live &= live - 1;
            const uint32_t prof_i = __shfl_sync(0xFFFFFFFFu, q.y, j) & 0xFFu;
            if (prof_i >= prof.n) return depth;             // an unknown profile has no candidate
            const uint32_t pi = p.prio[rb + j];
            unsigned long long best = ~0ull;
            for (uint32_t g = lane; g < c; g += 32)
                best = min(best, pg_best(s_masks, tab[b0 + g], prof_i, pi, st.prio[b0 + g], st.occ[b0 + g], st.rs[b0 + g], base + b0 + g));
            const unsigned long long win = warp_min(best);  // every lane has read its bytes: the owner may rewrite one below
            if (win == ~0ull) return depth;
            mx = max(mx, (uint32_t)(win >> 42));
            sum += (uint32_t)(win >> 31) & 0x7FFu;
            cnt += (uint32_t)(win >> 27) & 0xFu;
            const uint32_t g = (uint32_t)(win >> 3) & 0xFFFFFFu;
            if (((g - base - b0) & 31u) == lane) {
                const uint32_t m = s_masks[((uint32_t)tab[g - base] * ISL_MAX_PROFILES + prof_i) * ISL_MAX_STARTS + ((uint32_t)win & 7u)];
                pg_take(p, prof, st, g - base, g, m, rb + j, commit);
            }
            __syncwarp();
            ++depth;
        }
    }
    *all = true;
    return depth;
}

// One gang of requests [r0, r1) of any-node or (distinct) distinct-node locality, every thread of the CTA (P3, P5: rule 4).  `rank`
// counts the ALLOC members that took a GPU; the one that found none stops the gang, and every CTA puts back, in reverse order, the
// logged GPUs of its share and reports their members GANG_ABORTED with an empty evict row.
__device__ __forceinline__ void pg_members(const PreemptArgs& p, const DevProfiles& prof, const NodeShare& sh,
                                           const PgState& live, const uint8_t* tab, uint8_t* mark, const uint8_t* s_masks, PgLog* log,
                                           uint32_t r0, uint32_t r1, bool distinct, uint32_t& parity, unsigned long long* s_warp,
                                           unsigned long long* s_win, uint32_t tid, uint32_t lane, uint32_t warp) {
    const uint32_t base = sh.base, cnt = sh.cnt;
    if (distinct) for (uint32_t g = tid; g < cnt; g += kGnThreads) mark[g] = 0;
    __syncthreads();                                        // also orders the previous gang's commits before this gang's reads
    uint32_t rank = 0;
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t y = p.in[r].y, pq = y & 0xFFu;
        if (((y >> 8) & 0xFFu) != ISL_OP_ALLOC) continue;
        unsigned long long win = ~0ull;                     // an unknown profile fails without a barrier: every CTA knows it
        if (pq < prof.n) {
            const uint32_t pi = p.prio[r];
            unsigned long long best = ~0ull;
            for (uint32_t g = tid; g < cnt; g += kGnThreads)
                if (!distinct || !mark[g]) best = min(best, pg_best(s_masks, tab[g], pq, pi, live.prio[g], live.occ[g], live.rs[g], base + g));
            win = grid_min<kGnThreads>(best, p.keys, parity, s_warp, s_win);
        }
        if (win == ~0ull) {
            cooperative_groups::this_grid().sync();         // every CTA's log entries of this gang are in L2
            if (tid == 0) {
                for (uint32_t k = rank; k-- > 0;) {
                    const uint32_t gw = __ldcg(&log[k].gw), pos = gw - base;
                    if (pos >= cnt) continue;
                    const uint32_t o_rs = __ldcg(&log[k].o_rs), rr = __ldcg(&log[k].r);
                    live.prio[pos] = __ldcg(&log[k].prio); live.occ[pos] = (uint8_t)o_rs; live.rs[pos] = (uint8_t)(o_rs >> 8);
                    p.out[rr] = pack_result(ISL_GPU_NONE, ISL_START_NONE, prof.rows[p.in[rr].y & 0xFFu].size, ISL_ST_GANG_ABORTED);
                    for (uint32_t j = 0; j < ISL_SLOTS; ++j) p.evict[(size_t)rr * ISL_SLOTS + j] = kVictimNone;
                }
            }
            if (blockIdx.x == 0 && warp == 0) abort_gang_members(p.in, p.out, prof, r, r1, 0, lane);
            return;
        }
        const uint32_t gw = (uint32_t)(win >> 3) & 0xFFFFFFu, pos = gw - base;
        if (pos < cnt) {                                    // this CTA owns the GPU
            if (tid == 0) {
                const PgLog e{live.prio[pos], r, gw, (uint32_t)live.occ[pos] | (uint32_t)live.rs[pos] << 8, 0u};
                log[rank] = e;
                const uint32_t m = s_masks[((uint32_t)tab[pos] * ISL_MAX_PROFILES + pq) * ISL_MAX_STARTS + ((uint32_t)win & 7u)];
                pg_take(p, prof, live, pos, gw, m, r, true);
            }
            if (distinct) {                                 // the member's node is used for the rest of the gang
                uint32_t jl = sh.j0, jh = sh.j1;            // nb(jl) <= base + pos < nb(jh): the last such jl is the non-empty node
                while (jh - jl > 1) {
                    const uint32_t mid = (jl + jh) / 2;
                    if (sh.nb(mid) - base <= pos) jl = mid; else jh = mid;
                }
                for (uint32_t g = sh.nb(jl) - base + tid; g < sh.nb(jl + 1) - base; g += kGnThreads) mark[g] = 1;
            }
        }
        __syncthreads();                                    // the owner's state and marks are in place before the next member's scan
        ++rank;
    }
}

// One gang of requests [r0, r1) of one-node locality, every thread of the CTA (P3, P5: G3).  Each warp evaluates nodes of the share on
// the scratch copy; a node's key is the two words (max + 1 << 31 | sum, count << 32 | node) for a node that takes the gang, else
// (gn_fail_key(depth, node), 0).  The first grid_min takes the least first word, the second the least second word among the CTAs that
// hold it.  The owner of the winning node replays the gang on its live state; a failure: CTA 0 reports every ALLOC member except the one
// at the deepest depth D GANG_ABORTED.
__device__ __forceinline__ void pg_one_node(const PreemptArgs& p, const DevProfiles& prof, const NodeShare& sh, const PgState& live,
                                            const PgState& scr, const uint8_t* tab, const uint8_t* s_masks, uint32_t r0, uint32_t r1,
                                            uint32_t& parity, unsigned long long* s_warp, unsigned long long* s_win, uint32_t lane,
                                            uint32_t warp) {
    __syncthreads();                                        // the previous gang's commits are in the live state before this gang's reads
    unsigned long long hi = ~0ull, lo = ~0ull;              // the least key of this warp's nodes
    for (uint32_t j = sh.j0 + warp; j < sh.j1; j += kGnThreads / 32) {
        const uint32_t b0 = sh.nb(j) - sh.base, c = sh.nb(j + 1) - sh.base - b0;
        if (c == 0) continue;                               // an empty node takes nothing: depth 0, the floor of every failure
        for (uint32_t g = lane; g < c; g += 32) {
            scr.prio[b0 + g] = live.prio[b0 + g]; scr.occ[b0 + g] = live.occ[b0 + g]; scr.rs[b0 + g] = live.rs[b0 + g];
        }
        __syncwarp();
        bool all;
        uint32_t mx, sum, cnt;
        const uint32_t d = pg_node_resolve(p, prof, scr, tab, s_masks, b0, c, sh.base, r0, r1, false, lane, &all, mx, sum, cnt);
        const unsigned long long kh = all ? ((unsigned long long)mx << 31) | sum : gn_fail_key(d, j);
        const unsigned long long kl = all ? ((unsigned long long)cnt << 32) | j : 0ull;
        if (kh < hi || (kh == hi && kl < lo)) { hi = kh; lo = kl; }
    }
    const unsigned long long win = grid_min<kGnThreads>(hi, p.keys, parity, s_warp, s_win);
    if (!(win & kGnFail)) {
        const uint32_t j = (uint32_t)grid_min<kGnThreads>(hi == win ? lo : ~0ull, p.keys, parity, s_warp, s_win);
        if (j >= sh.j0 && j < sh.j1 && warp == 0) {         // the owner replays the gang on its live state
            const uint32_t b0 = sh.nb(j) - sh.base, c = sh.nb(j + 1) - sh.base - b0;
            bool all;
            uint32_t mx, sum, cnt;
            pg_node_resolve(p, prof, live, tab, s_masks, b0, c, sh.base, r0, r1, true, lane, &all, mx, sum, cnt);
        }
    } else if (blockIdx.x == 0 && warp == 0) {              // the deepest failure's depth; ~0ull (no node evaluated) is depth 0 as well
        abort_gang_members(p.in, p.out, prof, r0, r1, gn_fail_depth(win), lane);
    }
}

// kLoc: ISL_GANG_ANY_NODES, _ONE_NODE or _DISTINCT_NODES for every gang, or kLocPerGang for each gang's byte (0, 1 or 3, checked on the
// host).  With a constant kLoc the compiler drops the other bodies.
template <uint32_t kLoc>
__global__ void __launch_bounds__(kGnThreads, 1) k_preempt_gangs(GangNodeArgs a, PreemptArgs p, DevProfiles prof, PgLog* log,
                                                                const uint8_t* __restrict__ locality) {
    extern __shared__ __align__(16) unsigned char pg_smem[];
    __shared__ uint8_t s_masks[kMaxTables * ISL_MAX_PROFILES * ISL_MAX_STARTS];
    __shared__ unsigned long long s_warp[kGnThreads / 32];
    __shared__ unsigned long long s_win;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const NodeShare sh(a, pg_smem);                         // a.share == 0: it copies nothing
    // p.per_cta: GPUs per array of a share in shared memory, 0 = every share's arrays in global memory, strided by the partition
    const size_t S = p.per_cta ? p.per_cta : p.Gr, off = p.per_cta ? 0 : sh.base;
    unsigned char* const mem = p.per_cta ? pg_smem : a.scratch;
    const PgState live{reinterpret_cast<unsigned long long*>(mem) + off, mem + 16 * S + off, mem + 17 * S + off};
    const PgState scr{reinterpret_cast<unsigned long long*>(mem) + S + off, mem + 19 * S + off, mem + 20 * S + off};
    uint8_t* const tab = mem + 18 * S + off;
    for (uint32_t i = tid; i < sizeof(s_masks); i += kGnThreads) s_masks[i] = p.masks[i];
    for (uint32_t g = tid; g < sh.cnt; g += kGnThreads) {
        const uint32_t gw = sh.base + g;
        const uint4* w4 = reinterpret_cast<const uint4*>(p.vmap + (size_t)gw * ISL_SLOTS);
        const uint4 w0 = w4[0], w1 = w4[1];
        const uint32_t w[ISL_SLOTS] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
        unsigned long long pr = 0;
        uint32_t rs = 0;
#pragma unroll
        for (uint32_t s = 0; s < ISL_SLOTS; ++s) {
            const uint32_t v = w[s] == kVictimNone ? 0xFFu : p.victims[w[s]].priority;
            pr |= (unsigned long long)v << (8 * s);
            if (w[s] != kVictimNone && (s == 0 || w[s - 1] != w[s])) rs |= 1u << s;
        }
        live.prio[g] = pr; live.rs[g] = (uint8_t)rs;
        live.occ[g] = p.occ[p.lo + gw]; tab[g] = p.gtab[p.lo + gw];
    }
    for (uint32_t i = blockIdx.x * kGnThreads + tid; i < p.n; i += gridDim.x * kGnThreads) {      // default records
        const uint32_t y = p.in[i].y, q = y & 0xFFu;
        p.out[i] = ((y >> 8) & 0xFFu) != ISL_OP_ALLOC ? pack_result(ISL_GPU_NONE, ISL_START_NONE, 0, ISL_ST_NOOP)
                   : q >= prof.n                      ? pack_result(ISL_GPU_NONE, ISL_START_NONE, 0, ISL_ST_BAD_PROFILE)
                                                      : pack_result(ISL_GPU_NONE, ISL_START_NONE, prof.rows[q].size, ISL_ST_NO_CAPACITY);
    }
    cooperative_groups::this_grid().sync();                 // the defaults are written before any owner or CTA 0 rewrites one
    uint32_t parity = 0;
    for (uint32_t gi = 0; gi < a.n_gangs; ++gi) {
        const uint32_t r0 = __ldg(a.gang_off + gi), r1 = __ldg(a.gang_off + gi + 1), loc = kLoc == kLocPerGang ? __ldg(locality + gi) : kLoc;
        if (loc == ISL_GANG_ONE_NODE)
            pg_one_node(p, prof, sh, live, scr, tab, s_masks, r0, r1, parity, s_warp, &s_win, lane, warp);
        else
            pg_members(p, prof, sh, live, tab, scr.occ, s_masks, log, r0, r1, loc == ISL_GANG_DISTINCT_NODES, parity, s_warp, &s_win, tid, lane,
                       warp);
    }
}

}  // namespace isl
