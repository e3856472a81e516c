// gang_min_fast.cpp — brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_MIN_MEMBERS engine (include/islplace.h, rules
// M1-M7) on flat occupancy bytes, for all four localities.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_ganglocal<per_gang, min_members> and the single-core CPU baseline of
// tools/gang_min_time.py.  Every FREE of the call is applied first; then, gang after gang, the gang's locality is run on a copy of the
// occupancy until it commits or stops at ALLOC member f: 0 member by member over every GPU of the range, 1 every node in scan order with
// the first deepest node kept, 2 rounds of that, 3 member by member over the GPUs of nodes the gang does not use yet.  A gang that commits,
// or stops at f >= m', keeps the copy and its first f records; any other gang drops it.  It shares nothing with the kernel or with the
// other brute forces but the rules.
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

struct Call {
    uint32_t n_nodes, n_profiles, quirks, policy, lo, hi;
    const uint32_t* node_off;
    const uint8_t* node_table;
    const isl_profile* rows;
    std::vector<uint32_t> node_of;          // the node of every GPU
    std::vector<int16_t> memo;              // [table][profile][byte]: min-frag scores, -1 until first asked; empty: no memo

    bool descending() const { return policy == ISL_POLICY_RIGHT_TO_LEFT; }

    // the first legal start of profile p on byte o of a node of table t, in row order: its mask, 0 for none
    uint32_t fit(uint32_t t, uint32_t p, uint32_t o) const {
        const isl_profile& row = rows[(size_t)t * n_profiles + p];
        for (uint32_t k = 0; k < row.n_starts; ++k) {
            const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
            if (m && !(o & m)) return m;
        }
        return 0;
    }

    // what the policy minimises when profile p takes `mine` on byte o of a node of table t (first-fit family: nothing)
    uint32_t score(uint32_t t, uint32_t p, uint32_t o, uint32_t mine) {
        if (policy == ISL_POLICY_BEST_FIT) return 8u - (uint32_t)__builtin_popcount(o | mine);
        if (policy != ISL_POLICY_MIN_FRAG) return 0;
        int16_t* s = memo.empty() ? nullptr : &memo[((size_t)t * n_profiles + p) * 256 + o];
        if (s && *s >= 0) return (uint32_t)*s;
        uint32_t lost = 0;                  // (profile, start) pairs of the node's table that stop being feasible
        for (uint32_t q = 0; q < n_profiles; ++q) {
            const isl_profile& row = rows[(size_t)t * n_profiles + q];
            for (uint32_t k = 0; k < row.n_starts; ++k) {
                const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
                lost += m && !(o & m) && ((o | mine) & m);
            }
        }
        if (s) *s = (int16_t)lost;
        return lost;
    }

    // places profile p on the best GPU of [a, b) (scan order, ties to the first) whose node `used` does not mark, on `bytes`
    // (bytes[g - base] is GPU g); false when no GPU admits it
    bool place(uint8_t* bytes, uint32_t base, uint32_t a, uint32_t b, uint32_t p, const std::vector<uint8_t>* used, isl_result& rec) {
        if (p >= n_profiles) return false;
        bool found = false;
        uint32_t best_g = 0, best_m = 0, best_s = 0;
        for (uint32_t k = 0; k < b - a; ++k) {
            const uint32_t g = descending() ? b - 1 - k : a + k;
            if (used && (*used)[node_of[g]]) continue;
            const uint32_t t = node_table[node_of[g]], m = fit(t, p, bytes[g - base]);
            if (!m) continue;
            const uint32_t sc = score(t, p, bytes[g - base], m);
            if (!found || sc < best_s) { found = true; best_g = g; best_m = m; best_s = sc; }
        }
        if (!found) return false;
        bytes[best_g - base] |= (uint8_t)best_m;
        rec = {best_g, (uint8_t)__builtin_ctz(best_m), (uint8_t)__builtin_popcount(best_m), (uint16_t)ISL_ST_PLACED};
        return true;
    }

    // the GPUs of node v inside the range
    uint32_t first(uint32_t v) const { return std::min(std::max(node_off[v], lo), hi); }
    uint32_t last(uint32_t v) const { return std::min(std::max(node_off[v + 1], lo), hi); }

    // members[from..] on node v, whose bytes are `bytes`, in order, until one does not fit: how many fit
    size_t run_node(std::vector<uint8_t>& bytes, uint32_t v, const std::vector<uint32_t>& profile, size_t from, std::vector<isl_result>& rec) {
        size_t k = from;
        while (k < profile.size() && place(bytes.data(), first(v), first(v), last(v), profile[k], nullptr, rec[k])) ++k;
        return k - from;
    }

    // one locality's rules on `work` (the occupancy, updated with what the run placed): how many leading members it placed, f
    size_t run(uint32_t loc, std::vector<uint8_t>& work, const std::vector<uint32_t>& profile, std::vector<isl_result>& rec) {
        const size_t k = profile.size();
        if (loc == ISL_GANG_ANY_NODES || loc == ISL_GANG_DISTINCT_NODES) {      // rules 2-4 / S2-S3, member by member
            std::vector<uint8_t> used(n_nodes, 0);
            size_t f = 0;
            for (; f < k; ++f) {
                if (!place(work.data(), 0, lo, hi, profile[f], loc == ISL_GANG_DISTINCT_NODES ? &used : nullptr, rec[f])) break;
                used[node_of[rec[f].gpu]] = 1;
            }
            return f;
        }
        size_t f = 0;                                   // G2-G3 (one round) / F2-F3 (rounds)
        for (;;) {
            size_t best_d = 0;
            uint32_t best_v = 0;
            std::vector<uint8_t> best_bytes;
            std::vector<isl_result> best_rec(rec.size()), r(rec.size());
            for (uint32_t s = 0; s < n_nodes; ++s) {
                const uint32_t v = descending() ? n_nodes - 1 - s : s;
                if (first(v) == last(v)) continue;
                std::vector<uint8_t> bytes(work.begin() + first(v), work.begin() + last(v));
                const size_t d = run_node(bytes, v, profile, f, r);
                if (d > best_d) { best_d = d; best_v = v; best_bytes.swap(bytes); best_rec.swap(r); }     // a tie keeps the first node
            }
            if (best_d == 0) return f;
            std::copy(best_bytes.begin(), best_bytes.end(), work.begin() + first(best_v));
            std::copy(best_rec.begin() + f, best_rec.begin() + f + best_d, rec.begin() + f);
            f += best_d;
            if (f == k || loc == ISL_GANG_ONE_NODE) return f;
        }
    }
};

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off [n_nodes + 1] and node_table [n_nodes] in canonical order; occ: G bytes (canonical order), updated
// in place; default_size[p]: the size an unplaced ALLOC reports; [lo, hi): the canonical range (the engine's partition); memo: remember
// every min-frag score per (table, profile, byte).  locality[gang] (ISL_GANG_*) and min_members[gang] (m', M1) per gang.  out as
// isl_place_gangs writes it.  Returns the members placed (stats.placed).
uint64_t gmf_place_gangs(uint32_t n_nodes, const uint32_t* node_off, const uint8_t* node_table, uint32_t n_profiles, const isl_profile* rows,
                         const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy,
                         uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out, uint32_t memo,
                         const uint8_t* locality, const uint32_t* min_members) {
    Call c{n_nodes, n_profiles, quirks, policy, lo, hi, node_off, node_table, rows, {}, {}};
    const uint32_t G = node_off[n_nodes], n = gang_off[n_gangs];
    c.node_of.resize(G);
    for (uint32_t v = 0; v < n_nodes; ++v) for (uint32_t g = node_off[v]; g < node_off[v + 1]; ++g) c.node_of[g] = v;
    if (memo && policy == ISL_POLICY_MIN_FRAG)
        c.memo.assign((size_t)(*std::max_element(node_table, node_table + n_nodes) + 1) * n_profiles * 256, -1);
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
    uint64_t placed = 0;
    std::vector<uint8_t> work(occ, occ + G);
    for (uint32_t gi = 0; gi < n_gangs; ++gi) {
        std::vector<uint32_t> members, profile;         // the gang's ALLOCs in order and their profiles
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1]; ++i)
            if (in[i].op == ISL_OP_ALLOC) { members.push_back(i); profile.push_back(in[i].profile); }
        if (members.empty()) continue;
        std::vector<isl_result> rec(members.size());
        const size_t k = members.size(), f = c.run(locality[gi], work, profile, rec);
        const bool commit = f == k || f >= min_members[gi];     // M2 / M3
        for (size_t q = 0; q < k; ++q) {
            const uint32_t p = profile[q];
            const isl_result unplaced{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)(p < n_profiles ? default_size[p] : 0), 0};
            if (q < f && commit) out[members[q]] = rec[q];
            else if (q != f) {                          // member f keeps its record
                out[members[q]] = unplaced;
                out[members[q]].status = (uint16_t)(commit ? ISL_ST_GANG_TRIMMED : ISL_ST_GANG_ABORTED);
            }
        }
        for (size_t q = 0; q < f; ++q) {                // only the GPUs of the run's placements changed
            const uint32_t g = rec[q].gpu;
            if (commit) occ[g] = work[g];
            else work[g] = occ[g];                      // rule 5 / M4
        }
        if (commit) placed += f;
    }
    return placed;
}

}  // extern "C"
