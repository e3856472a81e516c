// gang_few_fast.cpp — brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_FEW_NODES engine (include/islplace.h, rules F1-F6)
// on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_ganglocal<few_nodes> and the single-core CPU baseline of tools/gang_few_time.py.  Every
// FREE of the call is applied first; then, gang after gang, round after round, every node of the range is simulated in scan order on a copy
// of its bytes, resolving the remaining ALLOC members one by one, each scoring every GPU of the node that admits it.  The node that places
// the most leading members (the first in scan order on a tie) keeps its copy; a round in which no node places one aborts the gang and drops
// every copy kept so far.  It shares nothing with the kernel but the rules.
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

struct Ctx {
    uint32_t n_profiles, quirks, policy;
    const isl_profile* rows;
    std::vector<int16_t> memo;              // [table][profile][byte]: a member's score, -1 until first asked; empty: no memo
};

// what the policy minimises on byte o for a placement of mask `mine` of profile p on a node of table t (first-fit family: nothing)
uint32_t score(const Ctx& c, uint32_t t, uint32_t o, uint32_t mine) {
    if (c.policy == ISL_POLICY_BEST_FIT) return 8u - (uint32_t)__builtin_popcount(o | mine);
    if (c.policy != ISL_POLICY_MIN_FRAG) return 0;
    uint32_t lost = 0;                      // (profile, start) pairs of the node's table that stop being feasible
    for (uint32_t q = 0; q < c.n_profiles; ++q) {
        const isl_profile& row = c.rows[(size_t)t * c.n_profiles + q];
        for (uint32_t k = 0; k < row.n_starts; ++k) {
            const uint32_t m = legal_mask(row.size, row.starts[k], c.quirks);
            lost += m && !(o & m) && ((o | mine) & m);
        }
    }
    return lost;
}

uint32_t member_score(Ctx& c, uint32_t t, uint32_t p, uint32_t o, uint32_t mine) {
    if (c.memo.empty()) return score(c, t, o, mine);
    int16_t& s = c.memo[((size_t)t * c.n_profiles + p) * 256 + o];
    if (s < 0) s = (int16_t)score(c, t, o, mine);
    return (uint32_t)s;
}

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off [n_nodes + 1] and node_table [n_nodes] in canonical order; occ: G bytes (canonical order), updated
// in place; default_size[p]: the size an unplaced ALLOC reports; [lo, hi): the canonical range (the engine's partition); memo: remember
// every score per (table, profile, byte).  out as isl_place_gangs writes it.  rounds (may be NULL): per request, the round (from 0) that
// placed it in a committed gang, else -1.
void gff_place_gangs(uint32_t n_nodes, const uint32_t* node_off, const uint8_t* node_table, uint32_t n_profiles, const isl_profile* rows,
                     const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy,
                     uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out, uint32_t memo, int32_t* rounds) {
    Ctx c{n_profiles, quirks, policy, rows, {}};
    if (memo && policy == ISL_POLICY_MIN_FRAG)
        c.memo.assign((size_t)(*std::max_element(node_table, node_table + n_nodes) + 1) * n_profiles * 256, -1);
    const uint32_t G = node_off[n_nodes], n = gang_off[n_gangs];
    const bool descending = policy == ISL_POLICY_RIGHT_TO_LEFT;
    for (uint32_t i = 0; i < n; ++i) {                  // rule 1: every FREE first; default records for the rest
        const isl_request& r = in[i];
        if (rounds) rounds[i] = -1;
        if (r.op == ISL_OP_FREE) {
            const bool ok = r.handle < G && r.size > 0 && r.start + r.size <= 8;
            if (ok && r.handle >= lo && r.handle < hi) occ[r.handle] &= (uint8_t)~(((1u << r.size) - 1u) << r.start);
            out[i] = {r.handle, r.start, r.size, (uint16_t)(ok ? ISL_ST_FREED : ISL_ST_BAD_SPAN)};
        } else if (r.op == ISL_OP_ALLOC) {
            out[i] = r.profile < n_profiles ? isl_result{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, default_size[r.profile], (uint16_t)ISL_ST_NO_CAPACITY}
                                            : isl_result{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_BAD_PROFILE};
        } else out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP};
    }
    std::vector<uint8_t> work(occ, occ + G);            // the occupancy with this gang's earlier rounds
    for (uint32_t gi = 0; gi < n_gangs; ++gi) {
        std::vector<uint32_t> members;                  // the gang's ALLOCs in order
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1]; ++i) if (in[i].op == ISL_OP_ALLOC) members.push_back(i);
        if (members.empty()) continue;
        std::vector<isl_result> rec(members.size());
        std::vector<int32_t> round_of(members.size(), -1);
        std::vector<std::pair<uint32_t, uint32_t>> touched;     // the GPU ranges of the nodes the rounds used
        size_t m = 0;                                   // F2: the first member not placed yet
        for (int32_t round = 0; m < members.size(); ++round) {
            size_t best_d = 0;
            uint32_t best_a = 0;
            std::vector<uint8_t> best_bytes;
            std::vector<isl_result> best_placed;
            for (uint32_t s = 0; s < n_nodes; ++s) {
                const uint32_t node = descending ? n_nodes - 1 - s : s;
                const uint32_t a = std::max(node_off[node], lo), b = std::min(node_off[node + 1], hi);
                if (a >= b) continue;
                std::vector<uint8_t> bytes(work.begin() + a, work.begin() + b);     // bytes[g - a] is GPU g
                std::vector<isl_result> placed;
                for (size_t k = m; k < members.size(); ++k) {
                    const uint32_t p = in[members[k]].profile;
                    if (p >= n_profiles) break;
                    const isl_profile& row = rows[(size_t)node_table[node] * n_profiles + p];
                    bool found = false;
                    uint32_t best_g = 0, best_m = 0, best_s = 0;
                    for (uint32_t q = 0; q < b - a; ++q) {     // the node's GPUs in scan order
                        const uint32_t g = descending ? b - 1 - q : a + q;
                        const uint32_t mk = first_mask(row, bytes[g - a], quirks);
                        if (!mk) continue;
                        const uint32_t sc = member_score(c, node_table[node], p, bytes[g - a], mk);
                        if (!found || sc < best_s) { found = true; best_g = g; best_m = mk; best_s = sc; }
                    }
                    if (!found) break;
                    bytes[best_g - a] |= (uint8_t)best_m;
                    placed.push_back({best_g, (uint8_t)__builtin_ctz(best_m), (uint8_t)__builtin_popcount(best_m), (uint16_t)ISL_ST_PLACED});
                }
                if (placed.size() > best_d) {            // strictly more: a tie keeps the earlier node in scan order
                    best_d = placed.size(); best_a = a; best_bytes.swap(bytes); best_placed.swap(placed);
                }
            }
            if (best_d == 0) break;                     // F3
            std::copy(best_bytes.begin(), best_bytes.end(), work.begin() + best_a);
            touched.emplace_back(best_a, best_a + (uint32_t)best_bytes.size());
            for (size_t k = 0; k < best_d; ++k) { rec[m + k] = best_placed[k]; round_of[m + k] = round; }
            m += best_d;
        }
        if (m == members.size()) {                      // the gang commits
            for (size_t k = 0; k < members.size(); ++k) {
                out[members[k]] = rec[k];
                if (rounds) rounds[members[k]] = round_of[k];
            }
            for (auto& t : touched) std::copy(work.begin() + t.first, work.begin() + t.second, occ + t.first);
            continue;
        }
        for (auto& t : touched) std::copy(occ + t.first, occ + t.second, work.begin() + t.first);     // rule 5: drop every round
        for (size_t k = 0; k < members.size(); ++k) {   // F3: member m keeps its record
            if (k == m) continue;
            const uint32_t p = in[members[k]].profile;
            out[members[k]] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)(p < n_profiles ? default_size[p] : 0), (uint16_t)ISL_ST_GANG_ABORTED};
        }
    }
}

}  // extern "C"
