// gang_node_fast.cpp — brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_ONE_NODE engine (include/islplace.h, rules G1-G6)
// on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_ganglocal<one_node> and the single-core CPU baseline of tools/gang_node_time.py.  Every
// FREE of the call is applied first; then, gang after gang, every node of the range is tried in scan order by resolving the gang's ALLOC
// members one by one on a copy of the node's bytes, each member scoring every GPU of the node that admits it.  The first node that takes
// every member is committed; without one, the deepest failure decides the record.  It shares nothing with the kernel but the rules.
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

// score() of profile p taking `mine`, its first legal start on byte o of a node of table t; with the memo on, each (table, profile, byte)
// is walked once, the first time a member asks for it
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
// every score per (table, profile, byte).  out as isl_place_gangs writes it.
void gnf_place_gangs(uint32_t n_nodes, const uint32_t* node_off, const uint8_t* node_table, uint32_t n_profiles, const isl_profile* rows,
                     const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy,
                     uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out, uint32_t memo) {
    Ctx c{n_profiles, quirks, policy, rows, {}};
    if (memo && policy == ISL_POLICY_MIN_FRAG)
        c.memo.assign((size_t)(*std::max_element(node_table, node_table + n_nodes) + 1) * n_profiles * 256, -1);
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
    for (uint32_t gi = 0; gi < n_gangs; ++gi) {
        std::vector<uint32_t> members;                  // the gang's ALLOCs in order
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1]; ++i) if (in[i].op == ISL_OP_ALLOC) members.push_back(i);
        if (members.empty()) continue;
        uint32_t deepest = 0;
        bool done = false;
        for (uint32_t s = 0; s < n_nodes && !done; ++s) {
            const uint32_t node = descending ? n_nodes - 1 - s : s;
            const uint32_t a = std::max(node_off[node], lo), b = std::min(node_off[node + 1], hi);
            if (a >= b) continue;
            std::vector<uint8_t> bytes(occ + a, occ + b);    // a copy of the node's bytes inside the range; bytes[g - a] is GPU g
            std::vector<isl_result> placed;
            for (uint32_t i : members) {
                const uint32_t p = in[i].profile;
                if (p >= n_profiles) break;
                const isl_profile& row = rows[(size_t)node_table[node] * n_profiles + p];
                bool found = false;
                uint32_t best_g = 0, best_m = 0, best_s = 0;
                for (uint32_t k = 0; k < b - a; ++k) {       // the node's GPUs in scan order
                    const uint32_t g = descending ? b - 1 - k : a + k;
                    const uint32_t m = first_mask(row, bytes[g - a], quirks);
                    if (!m) continue;
                    const uint32_t sc = member_score(c, node_table[node], p, bytes[g - a], m);
                    if (!found || sc < best_s) { found = true; best_g = g; best_m = m; best_s = sc; }
                }
                if (!found) break;
                bytes[best_g - a] |= (uint8_t)best_m;
                placed.push_back({best_g, (uint8_t)__builtin_ctz(best_m), (uint8_t)__builtin_popcount(best_m), (uint16_t)ISL_ST_PLACED});
            }
            if (placed.size() == members.size()) {      // G2: the first node that takes the whole gang
                for (size_t k = 0; k < members.size(); ++k) out[members[k]] = placed[k];
                memcpy(occ + a, bytes.data(), b - a);
                done = true;
            }
            deepest = std::max<uint32_t>(deepest, (uint32_t)placed.size());
        }
        if (done) continue;
        for (size_t k = 0; k < members.size(); ++k) {  // G3: the member at the deepest failure keeps its record
            if (k == deepest) continue;
            const uint32_t p = in[members[k]].profile;
            out[members[k]] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)(p < n_profiles ? default_size[p] : 0), (uint16_t)ISL_ST_GANG_ABORTED};
        }
    }
}

}  // extern "C"
