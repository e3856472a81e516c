// gang_score_all_fast.cpp — brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_NODE_SCORE_ALL
// engine (include/islplace.h, rules N1-N8 and C1-C8, with M1-M7 when the caller passes minima) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of the node-scored k_ganglocal instantiations of every gang kind and the single-core CPU
// baseline of tools/gang_score_all_time.py.  Every FREE of the call is applied first; then, gang after gang, the gang's locality is run
// on a copy of the occupancy until it commits or stops at ALLOC member f.  Every node is scored from the copy's bytes (cap = width x GPUs
// inside the range, busy = the bytes' slices under the width), and inside a node a member takes the first admitting GPU at its first
// legal start:
//   0        member by member, the best-scored node that admits the member, ties to the lowest node;
//   3        the same over the nodes the gang does not use yet;
//   4..255   the same over the nodes whose count of the gang's members is at most mu + byte - 4, mu the least count over the nodes that
//            admit the member;
//   1        every node resolves the members on a copy of its bytes; the deepest node wins, then the best score for the slices of the
//            members it placed, then the lowest node (one round);
//   2        rounds of that until every member is placed or the deepest node places none.
// A gang that commits, or stops at f >= m', keeps the copy and its first f records; any other gang drops it.  It shares nothing with the
// kernel or with the other brute forces but the rules.
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
    std::vector<uint32_t> width;            // node-scoring rule 2 per table

    // the first legal start of profile p on byte o of a node of table t, in row order: its mask, 0 for none
    uint32_t fit(uint32_t t, uint32_t p, uint32_t o) const {
        const isl_profile& row = rows[(size_t)t * n_profiles + p];
        for (uint32_t k = 0; k < row.n_starts; ++k) {
            const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
            if (m && !(o & m)) return m;
        }
        return 0;
    }
    uint32_t size(uint32_t v, uint32_t p) const { return rows[(size_t)node_table[v] * n_profiles + p].size; }

    // the GPUs of node v inside the range
    uint32_t first(uint32_t v) const { return std::min(std::max(node_off[v], lo), hi); }
    uint32_t last(uint32_t v) const { return std::min(std::max(node_off[v + 1], lo), hi); }

    // node-scoring rule 3 for node v on `bytes` (bytes[g] is GPU g) with req more slices: higher is better
    int64_t score(const std::vector<uint8_t>& bytes, uint32_t v, uint64_t req) const {
        const uint32_t w = width[node_table[v]];
        uint64_t busy = 0;
        for (uint32_t g = first(v); g < last(v); ++g) busy += __builtin_popcount(bytes[g] & ((1u << w) - 1u));
        const uint64_t cap = (uint64_t)w * (last(v) - first(v));
        return policy == ISL_POLICY_MOST_ALLOCATED ? (int64_t)(100 * (busy + req) / cap) : (int64_t)(100 * (cap - busy - req) / cap);
    }

    // profile p on node v's first admitting GPU of `b` (b[g - base] is GPU g): false when none admits it
    bool place_on(uint8_t* b, uint32_t base, uint32_t v, uint32_t p, isl_result& rec) const {
        for (uint32_t g = first(v); g < last(v); ++g) {
            const uint32_t m = fit(node_table[v], p, b[g - base]);
            if (!m) continue;
            b[g - base] |= (uint8_t)m;
            rec = {g, (uint8_t)__builtin_ctz(m), (uint8_t)__builtin_popcount(m), (uint16_t)ISL_ST_PLACED};
            return true;
        }
        return false;
    }
    bool admits(const std::vector<uint8_t>& bytes, uint32_t v, uint32_t p) const {
        for (uint32_t g = first(v); g < last(v); ++g) if (fit(node_table[v], p, bytes[g])) return true;
        return false;
    }

    // one locality's rules on `work` (the occupancy, updated with what the run placed): how many leading members it placed, f
    size_t run(uint32_t loc, std::vector<uint8_t>& work, const std::vector<uint32_t>& profile, std::vector<isl_result>& rec) const {
        const size_t k = profile.size();
        if (loc != ISL_GANG_ONE_NODE && loc != ISL_GANG_FEW_NODES) {      // N3, N4, C6: member by member
            std::vector<uint32_t> cnt(n_nodes, 0);
            size_t f = 0;
            for (; f < k; ++f) {
                const uint32_t p = profile[f];
                if (p >= n_profiles) break;
                uint64_t mu = UINT64_MAX;                // balanced: the least count over the nodes that admit the member
                if (loc > ISL_GANG_DISTINCT_NODES)
                    for (uint32_t v = 0; v < n_nodes; ++v)
                        if (first(v) < last(v) && admits(work, v, p)) mu = std::min<uint64_t>(mu, cnt[v]);
                int64_t best = -1;
                uint32_t best_v = 0;
                for (uint32_t v = 0; v < n_nodes; ++v) {
                    if (first(v) == last(v) || !admits(work, v, p)) continue;
                    if (loc == ISL_GANG_DISTINCT_NODES && cnt[v]) continue;
                    if (loc > ISL_GANG_DISTINCT_NODES && cnt[v] > mu + (loc - ISL_GANG_DISTINCT_NODES) - 1) continue;
                    const int64_t s = score(work, v, size(v, p));
                    if (s > best) { best = s; best_v = v; }                // a tie keeps the lower node
                }
                if (best < 0) break;
                place_on(work.data(), 0, best_v, p, rec[f]);
                ++cnt[best_v];
            }
            return f;
        }
        size_t f = 0;                                   // N5 / C4 / C5: rounds; one node stops after the first
        for (;;) {
            size_t best_d = 0;
            int64_t best_s = -1;
            std::vector<isl_result> best_rec(k), r(k);
            for (uint32_t v = 0; v < n_nodes; ++v) {
                if (first(v) == last(v)) continue;
                std::vector<uint8_t> bytes(work.begin() + first(v), work.begin() + last(v));
                size_t d = 0;
                uint64_t R = 0;
                while (f + d < k && profile[f + d] < n_profiles && place_on(bytes.data(), first(v), v, profile[f + d], r[f + d]))
                    R += size(v, profile[f + d++]);
                if (d == 0) continue;
                const int64_t s = score(work, v, R);
                if (d > best_d || (d == best_d && s > best_s)) { best_d = d; best_s = s; best_rec.swap(r); }     // ties: the lower node
            }
            if (best_d == 0) return f;
            for (size_t q = f; q < f + best_d; ++q) {
                rec[q] = best_rec[q];
                work[rec[q].gpu] |= (uint8_t)(((1u << rec[q].size) - 1u) << rec[q].start);
            }
            f += best_d;
            if (f == k || loc == ISL_GANG_ONE_NODE) return f;
        }
    }
};

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off [n_nodes + 1] and node_table [n_nodes] in canonical order; occ: G bytes (canonical order), updated
// in place; default_size[p]: the size an unplaced ALLOC reports; [lo, hi): the canonical range (the engine's partition); policy:
// ISL_POLICY_MOST_ALLOCATED or _LEAST_ALLOCATED.  locality[gang] (0..255: the start byte of its ALLOC members under
// ISL_FLAG_GANG_LOCALITY, else the engine's locality) and min_members[gang] (m', M1; the gang's ALLOC count without
// ISL_FLAG_GANG_MIN_MEMBERS) per gang.  out as isl_place_gangs writes it.  Returns the members placed (stats.placed).
uint64_t gsa_place_gangs(uint32_t n_nodes, const uint32_t* node_off, const uint8_t* node_table, uint32_t n_profiles, const isl_profile* rows,
                         const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy,
                         uint32_t n_gangs, const uint32_t* gang_off, const isl_request* in, isl_result* out, const uint8_t* locality,
                         const uint32_t* min_members) {
    Call c{n_nodes, n_profiles, quirks, policy, lo, hi, node_off, node_table, rows, {}};
    const uint32_t G = node_off[n_nodes], n = gang_off[n_gangs];
    c.width.assign(*std::max_element(node_table, node_table + n_nodes) + 1u, 0);
    for (uint32_t t = 0; t < c.width.size(); ++t)       // node-scoring rule 2: the largest start + size of the table's rows
        for (uint32_t p = 0; p < n_profiles; ++p) {
            const isl_profile& row = rows[(size_t)t * n_profiles + p];
            for (uint32_t k = 0; k < row.n_starts; ++k) c.width[t] = std::max<uint32_t>(c.width[t], row.starts[k] + row.size);
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
