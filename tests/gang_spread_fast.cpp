// gang_spread_fast.cpp — brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_DISTINCT_NODES engine (include/islplace.h, rules
// S1-S6) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_gangspread and the single-core CPU baseline of tools/gang_spread_time.py.  Every FREE
// of the call is applied first; then, gang after gang, the ALLOC members are resolved one by one: every GPU of the range, in scan order,
// whose node holds no earlier member of the gang is scored, the best one is taken on a copy of the bytes, and its node is added to the
// gang's used set.  A member with no GPU aborts the gang and the copy is dropped.  It shares nothing with the kernel but the rules.
#include <algorithm>
#include <cstdint>
#include <cstring>
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

// the first legal start of `row` on byte o, in row order: its mask, 0 for none
uint32_t first_mask(const isl_profile& row, uint32_t o, uint32_t quirks) {
    for (uint32_t k = 0; k < row.n_starts; ++k) {
        const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
        if (m && !(o & m)) return m;
    }
    return 0;
}

// what the policy minimises on byte o for a placement of mask `mine` of profile p on a node of table t (first-fit family: nothing)
uint32_t score(uint32_t policy, uint32_t n_profiles, const isl_profile* rows, uint32_t quirks, uint32_t t, uint32_t o, uint32_t mine) {
    if (policy == ISL_POLICY_BEST_FIT) return 8u - (uint32_t)__builtin_popcount(o | mine);
    if (policy != ISL_POLICY_MIN_FRAG) return 0;
    uint32_t lost = 0;                      // (profile, start) pairs of the node's table that stop being feasible
    for (uint32_t q = 0; q < n_profiles; ++q) {
        const isl_profile& row = rows[(size_t)t * n_profiles + q];
        for (uint32_t k = 0; k < row.n_starts; ++k) {
            const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
            lost += m && !(o & m) && ((o | mine) & m);
        }
    }
    return lost;
}

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off [n_nodes + 1] and node_table [n_nodes] in canonical order; occ: G bytes (canonical order), updated
// in place; default_size[p]: the size an unplaced ALLOC reports; [lo, hi): the canonical range (the engine's partition).  out as
// isl_place_gangs writes it.
void gsf_place_gangs(uint32_t n_nodes, const uint32_t* node_off, const uint8_t* node_table, uint32_t n_profiles, const isl_profile* rows,
                     const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy,
                     uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out) {
    const uint32_t G = node_off[n_nodes], n = gang_off[n_gangs];
    const bool descending = policy == ISL_POLICY_RIGHT_TO_LEFT;
    for (uint32_t i = 0; i < n; ++i) {                  // rule 1: every FREE first; default records for the rest
        const isl_request& r = in[i];
        if (r.op == ISL_OP_FREE) {
            const bool ok = r.handle < G && r.size > 0 && r.start + r.size <= 8;
            if (ok && r.handle >= lo && r.handle < hi) occ[r.handle] &= (uint8_t)~(((1u << r.size) - 1u) << r.start);
            out[i] = {r.handle, r.start, r.size, (uint16_t)(ok ? ISL_ST_FREED : ISL_ST_BAD_SPAN)};
        } else if (r.op == ISL_OP_ALLOC) {
            out[i] = r.profile < n_profiles ? isl_result{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, default_size[r.profile], (uint16_t)ISL_ST_NO_CAPACITY}
                                            : isl_result{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_BAD_PROFILE};
        } else out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP};
    }
    std::vector<uint32_t> node_of(G);                   // the node of every GPU
    for (uint32_t v = 0; v < n_nodes; ++v) for (uint32_t g = node_off[v]; g < node_off[v + 1]; ++g) node_of[g] = v;
    std::vector<uint8_t> used(n_nodes, 0);
    for (uint32_t gi = 0; gi < n_gangs; ++gi) {
        std::vector<uint32_t> members, nodes;           // the gang's ALLOCs in order; the nodes its placed members use
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1]; ++i) if (in[i].op == ISL_OP_ALLOC) members.push_back(i);
        std::vector<isl_result> placed;
        std::vector<uint8_t> bytes(occ + lo, occ + hi);     // the gang's tentative occupancy; bytes[g - lo] is GPU g
        for (uint32_t i : members) {
            const uint32_t p = in[i].profile;
            if (p >= n_profiles) break;
            bool found = false;
            uint32_t best_g = 0, best_m = 0, best_s = 0;
            for (uint32_t k = 0; k < hi - lo; ++k) {    // the range's GPUs in scan order
                const uint32_t g = descending ? hi - 1 - k : lo + k;
                if (used[node_of[g]]) continue;
                const isl_profile& row = rows[(size_t)node_table[node_of[g]] * n_profiles + p];
                const uint32_t m = first_mask(row, bytes[g - lo], quirks);
                if (!m) continue;
                const uint32_t sc = score(policy, n_profiles, rows, quirks, node_table[node_of[g]], bytes[g - lo], m);
                if (!found || sc < best_s) { found = true; best_g = g; best_m = m; best_s = sc; }
            }
            if (!found) break;
            bytes[best_g - lo] |= (uint8_t)best_m;
            used[node_of[best_g]] = 1;
            nodes.push_back(node_of[best_g]);
            placed.push_back({best_g, (uint8_t)__builtin_ctz(best_m), (uint8_t)__builtin_popcount(best_m), (uint16_t)ISL_ST_PLACED});
        }
        for (uint32_t v : nodes) used[v] = 0;
        if (placed.size() == members.size()) {          // S1 / rule 3: the gang commits
            for (size_t k = 0; k < members.size(); ++k) out[members[k]] = placed[k];
            memcpy(occ + lo, bytes.data(), hi - lo);
            continue;
        }
        for (size_t k = 0; k < members.size(); ++k) {  // S3 / rule 4: the first member that found nothing keeps its record
            if (k == placed.size()) continue;
            const uint32_t p = in[members[k]].profile;
            out[members[k]] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)(p < n_profiles ? default_size[p] : 0), (uint16_t)ISL_ST_GANG_ABORTED};
        }
    }
}

}  // extern "C"
