// node_score_fast.cpp — brute-force restatement of ISL_POLICY_MOST_ALLOCATED / ISL_POLICY_LEAST_ALLOCATED (include/islplace.h, rules
// 1-7) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_nodefit and the single-core CPU baseline of tools/node_score_time.py.  For every
// ALLOC it walks every node and every GPU of the range, recounts cap, busy and the GPUs that admit the profile from the bytes, scores
// the node with the integer formulas and keeps the first best node; then the node's first admitting GPU takes the first legal start of
// the row.  It shares nothing with the kernel but the rules.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../include/islplace.h"

namespace {

// the start search's legality of one (size, start), restated from :343-383 with the two quirks (Q1 strict bound, Q2 powers of two)
uint32_t legal_mask(uint32_t size, uint32_t v, uint32_t quirks) {
    if (v >= 8 || size == 0 || size > 8) return 0;
    if (size == 1) return 1u << v;
    if ((quirks & ISL_QUIRK_POW2_ONLY) && size != 2 && size != 4 && size != 8) return 0;
    if ((quirks & ISL_QUIRK_STRICT_BOUND) ? v + size >= 8 : v + size > 8) return 0;
    return ((1u << size) - 1u) << v;
}

// first legal free start of `row` on byte o in row order, or 9
uint32_t first_start(const isl_profile& row, uint32_t o, uint32_t quirks) {
    for (uint32_t k = 0; k < row.n_starts; ++k) {
        const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
        if (m && !(o & m)) return row.starts[k];
    }
    return ISL_START_NONE;
}

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off: n_nodes + 1 offsets; node_table: table of every node; occ: G bytes, canonical order, updated in
// place; [lo, hi): the canonical range; default_size[p]: the size an unplaced ALLOC reports.  out: n records.
int ns_place(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows, const uint8_t* node_table,
             const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy, uint32_t n,
             const isl_request* in, isl_result* out) {
    const uint32_t G = node_off[n_nodes];
    std::vector<uint32_t> width(n_tables, 0);
    for (uint32_t t = 0; t < n_tables; ++t)
        for (uint32_t p = 0; p < n_profiles; ++p) {
            const isl_profile& row = rows[(size_t)t * n_profiles + p];
            for (uint32_t k = 0; k < row.n_starts; ++k) width[t] = std::max<uint32_t>(width[t], row.starts[k] + row.size);
        }
    for (uint32_t i = 0; i < n; ++i) {          // rule 5 and batch semantics: every FREE first
        if (in[i].op != ISL_OP_FREE) continue;
        const uint32_t g = in[i].handle;
        if (g >= G || in[i].size == 0 || in[i].start + in[i].size > 8) { out[i] = {g, in[i].start, in[i].size, (uint16_t)ISL_ST_BAD_SPAN}; continue; }
        if (g >= lo && g < hi) occ[g] &= (uint8_t)~(((1u << in[i].size) - 1u) << in[i].start);
        out[i] = {g, in[i].start, in[i].size, (uint16_t)ISL_ST_FREED};
    }
    uint32_t dead = 0;                          // profiles with no candidate: occupancy only grows after the FREEs, so they stay without one
    for (uint32_t i = 0; i < n; ++i) {
        if (in[i].op == ISL_OP_FREE) continue;
        if (in[i].op != ISL_OP_ALLOC) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP}; continue; }
        const uint32_t p = in[i].profile;
        if (p >= n_profiles) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_BAD_PROFILE}; continue; }
        if ((dead >> p) & 1u) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, default_size[p], (uint16_t)ISL_ST_NO_CAPACITY}; continue; }
        int64_t best_score = -1;
        uint32_t best_node = 0;
        for (uint32_t v = 0; v < n_nodes; ++v) {
            const uint32_t a = std::max(lo, node_off[v]), b = std::min(hi, node_off[v + 1]);
            if (a >= b) continue;
            const uint32_t t = node_table[v];
            const isl_profile& row = rows[(size_t)t * n_profiles + p];
            uint64_t cap = 0, busy = 0;
            bool cand = false;
            for (uint32_t g = a; g < b; ++g) {
                cap += width[t];
                busy += __builtin_popcount(occ[g] & ((1u << width[t]) - 1u));
                cand |= first_start(row, occ[g], quirks) != ISL_START_NONE;
            }
            if (!cand) continue;
            const uint64_t req = row.size;
            const int64_t score = policy == ISL_POLICY_MOST_ALLOCATED ? (int64_t)(100 * (busy + req) / cap) : (int64_t)(100 * (cap - busy - req) / cap);
            if (score > best_score) { best_score = score; best_node = v; }
        }
        if (best_score < 0) {
            dead |= 1u << p;
            out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, default_size[p], (uint16_t)ISL_ST_NO_CAPACITY};
            continue;
        }
        const isl_profile& row = rows[(size_t)node_table[best_node] * n_profiles + p];
        for (uint32_t g = std::max(lo, node_off[best_node]); g < std::min(hi, node_off[best_node + 1]); ++g) {
            const uint32_t s = first_start(row, occ[g], quirks);
            if (s == ISL_START_NONE) continue;
            occ[g] |= (uint8_t)legal_mask(row.size, s, quirks);
            out[i] = {g, (uint8_t)s, row.size, (uint16_t)ISL_ST_PLACED};
            break;
        }
    }
    return ISL_OK;
}

}  // extern "C"
