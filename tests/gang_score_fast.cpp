// gang_score_fast.cpp — brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE engine (include/islplace.h, rules
// N1-N8) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of the node-scored k_ganglocal instantiations and the single-core CPU baseline of
// tools/gang_score_time.py.  Every FREE of the call is applied first; then, gang after gang, by the gang's locality:
//   any node / distinct nodes  for every ALLOC member, every node of the range (distinct: not one the gang already uses) is scored from
//                              its bytes (cap, busy, whether a GPU admits the member), the first best node takes the member on its first
//                              admitting GPU; a member with no node aborts the gang and the bytes go back to what they were before it;
//   one node                   every node of the range resolves the members first-fit on a copy of its bytes; among the nodes that take
//                              them all, the first with the best score for the sum of the members' row sizes wins; else G3.
// It shares nothing with the kernel but the rules.
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

// NodeResourcesFit's integer score with MaxNodeScore 100 (node-scoring rule 3)
int64_t node_score(uint32_t policy, uint64_t cap, uint64_t busy, uint64_t req) {
    return policy == ISL_POLICY_MOST_ALLOCATED ? (int64_t)(100 * (busy + req) / cap) : (int64_t)(100 * (cap - busy - req) / cap);
}

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off [n_nodes + 1] and node_table [n_nodes] in canonical order; occ: G bytes (canonical order), updated
// in place; default_size[p]: the size an unplaced ALLOC reports; [lo, hi): the canonical range (the engine's partition); policy:
// ISL_POLICY_MOST_ALLOCATED or _LEAST_ALLOCATED; locality: ISL_GANG_ANY_NODES, _ONE_NODE or _DISTINCT_NODES for every gang, or 4 for
// each gang's own byte (ISL_FLAG_GANG_LOCALITY).  out as isl_place_gangs writes it; returns the members committed (stats.placed).
uint64_t gsf_place_gangs(uint32_t n_nodes, const uint32_t* node_off, const uint8_t* node_table, uint32_t n_profiles, const isl_profile* rows,
                         const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy,
                         uint32_t locality, uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out) {
    const uint32_t G = node_off[n_nodes], n = gang_off[n_gangs];
    std::vector<uint32_t> width(*std::max_element(node_table, node_table + n_nodes) + 1u, 0);
    for (uint32_t t = 0; t < width.size(); ++t)
        for (uint32_t p = 0; p < n_profiles; ++p) {
            const isl_profile& row = rows[(size_t)t * n_profiles + p];
            for (uint32_t k = 0; k < row.n_starts; ++k) width[t] = std::max<uint32_t>(width[t], row.starts[k] + row.size);
        }
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
    // cap and busy of node v inside the range, from the bytes `b` (canonical GPU g is b[g])
    auto usage = [&](const uint8_t* b, uint32_t v, uint64_t& cap, uint64_t& busy) {
        const uint32_t w = width[node_table[v]];
        cap = busy = 0;
        for (uint32_t g = std::max(lo, node_off[v]); g < std::min(hi, node_off[v + 1]); ++g) {
            cap += w;
            busy += __builtin_popcount(b[g] & ((1u << w) - 1u));
        }
    };
    uint64_t placed = 0;
    for (uint32_t gi = 0; gi < n_gangs; ++gi) {
        std::vector<uint32_t> members;                  // the gang's ALLOCs in order
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1]; ++i) if (in[i].op == ISL_OP_ALLOC) members.push_back(i);
        if (members.empty()) continue;
        const uint32_t loc = locality == 4 ? in[members[0]].start : locality;
        uint32_t fail = (uint32_t)members.size();       // the ALLOC member that keeps its record when the gang aborts
        if (loc == ISL_GANG_ONE_NODE) {                 // N5
            uint32_t deepest = 0;
            int64_t best_score = -1;
            std::vector<isl_result> best;
            for (uint32_t v = 0; v < n_nodes; ++v) {
                const uint32_t a = std::max(node_off[v], lo), b = std::min(node_off[v + 1], hi);
                if (a >= b) continue;
                std::vector<uint8_t> bytes(occ + a, occ + b);
                std::vector<isl_result> got;
                uint64_t R = 0;
                for (uint32_t i : members) {            // the reference's search restricted to the node: first admitting GPU, first start
                    const uint32_t p = in[i].profile;
                    if (p >= n_profiles) break;
                    const isl_profile& row = rows[(size_t)node_table[v] * n_profiles + p];
                    uint32_t g = a, m = 0;
                    for (; g < b && !(m = first_mask(row, bytes[g - a], quirks)); ++g) {}
                    if (!m) break;
                    bytes[g - a] |= (uint8_t)m;
                    got.push_back({g, (uint8_t)__builtin_ctz(m), row.size, (uint16_t)ISL_ST_PLACED});
                    R += row.size;
                }
                deepest = std::max<uint32_t>(deepest, (uint32_t)got.size());
                if (got.size() != members.size()) continue;
                uint64_t cap, busy;
                usage(occ, v, cap, busy);
                const int64_t s = node_score(policy, cap, busy, R);
                if (s > best_score) { best_score = s; best = got; }
            }
            if (best_score >= 0) {
                for (size_t k = 0; k < members.size(); ++k) {
                    out[members[k]] = best[k];
                    occ[best[k].gpu] |= (uint8_t)(((1u << best[k].size) - 1u) << best[k].start);
                }
            } else fail = deepest;
        } else {                                        // N3 / N4: member by member, on the live bytes, rolled back on a failure
            std::vector<uint8_t> before(occ + lo, occ + hi);
            std::vector<uint32_t> used;                 // nodes of the gang's earlier members (distinct nodes)
            for (uint32_t k = 0; k < members.size() && fail == members.size(); ++k) {
                const uint32_t i = members[k], p = in[i].profile;
                if (p >= n_profiles) { fail = k; break; }
                int64_t best_score = -1;
                uint32_t best_node = 0;
                for (uint32_t v = 0; v < n_nodes; ++v) {
                    const uint32_t a = std::max(node_off[v], lo), b = std::min(node_off[v + 1], hi);
                    if (a >= b) continue;
                    if (loc == ISL_GANG_DISTINCT_NODES && std::find(used.begin(), used.end(), v) != used.end()) continue;
                    const isl_profile& row = rows[(size_t)node_table[v] * n_profiles + p];
                    bool cand = false;
                    for (uint32_t g = a; g < b && !cand; ++g) cand = first_mask(row, occ[g], quirks) != 0;
                    if (!cand) continue;
                    uint64_t cap, busy;
                    usage(occ, v, cap, busy);
                    const int64_t s = node_score(policy, cap, busy, row.size);
                    if (s > best_score) { best_score = s; best_node = v; }
                }
                if (best_score < 0) { fail = k; break; }
                const isl_profile& row = rows[(size_t)node_table[best_node] * n_profiles + p];
                for (uint32_t g = std::max(lo, node_off[best_node]);; ++g) {
                    const uint32_t m = first_mask(row, occ[g], quirks);
                    if (!m) continue;
                    occ[g] |= (uint8_t)m;
                    out[i] = {g, (uint8_t)__builtin_ctz(m), row.size, (uint16_t)ISL_ST_PLACED};
                    break;
                }
                used.push_back(best_node);
            }
            if (fail != members.size()) memcpy(occ + lo, before.data(), before.size());     // rule 5
        }
        if (fail == members.size()) { placed += members.size(); continue; }
        for (size_t k = 0; k < members.size(); ++k) {   // rule 4 / G3: the member at `fail` keeps its record
            if (k == fail) continue;
            const uint32_t p = in[members[k]].profile;
            out[members[k]] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)(p < n_profiles ? default_size[p] : 0), (uint16_t)ISL_ST_GANG_ABORTED};
        }
    }
    return placed;
}

}  // extern "C"
