// first_available_fast.cpp — brute-force restatement of profile alternatives (ISL_FLAG_FIRST_AVAILABLE, include/islplace.h A1-A8) on
// flat occupancy bytes, for every policy.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_bestfit's and k_nodefit's pod loops and the single-core CPU baseline of
// tools/first_available_time.py.  For every ALLOC it tries the policy's rule over every GPU (or node) of the range from the bytes: the
// first admitting GPU in scan order (FIRST_FIT, RIGHT_TO_LEFT), the least score with ties to the lowest GPU (BEST_FIT, MIN_FRAG), or the
// best node score with ties to the lowest node and that node's first admitting GPU (MOST_ / LEAST_ALLOCATED).  Pods are found by
// comparing each request with the one before it.  It shares nothing with the kernels but the rules.
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

// the mask of the first legal free start of `row` on byte o in row order, or 0
uint32_t first_mask(const isl_profile& row, uint32_t o, uint32_t quirks) {
    for (uint32_t k = 0; k < row.n_starts; ++k) {
        const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
        if (m && !(o & m)) return m;
    }
    return 0;
}

struct Cluster {
    uint32_t G, n_nodes, n_profiles, quirks, policy, lo, hi;
    const uint32_t* node_off;
    const isl_profile* rows;        // [table][profile]
    const uint8_t* node_table;
    uint8_t* occ;
    std::vector<uint32_t> node_of;  // node of every GPU
    std::vector<uint32_t> width;    // per table: the largest start + size over its rows
    std::vector<std::vector<uint32_t>> cand;    // per table: every (profile, start) mask the search can return
    mutable std::vector<int32_t> memo;          // [table][profile][byte]: score << 8 | mask, -1 until first asked; empty: no memo

    const isl_profile& row(uint32_t g, uint32_t p) const { return rows[(size_t)node_table[node_of[g]] * n_profiles + p]; }

    // what the best-fit family minimises on GPU g for a placement `mine` (BEST_FIT: free slices after it; MIN_FRAG: the table's
    // (profile, start) pairs it makes infeasible)
    uint32_t score(uint32_t g, uint32_t mine) const {
        const uint32_t o = occ[g];
        if (policy == ISL_POLICY_BEST_FIT) return 8u - (uint32_t)__builtin_popcount(o | mine);
        uint32_t v = 0;
        for (uint32_t m : cand[node_table[node_of[g]]]) v += ((o & m) == 0) && (((o | mine) & m) != 0);
        return v;
    }

    // the best-fit family's (score, first legal mask) of profile p on GPU g as score << 8 | mask (mask 0: no legal start); with the memo
    // on, each (table, profile, byte) is walked once, the first time a GPU asks for it
    uint32_t scored(uint32_t g, uint32_t p) const {
        int32_t* v = memo.empty() ? nullptr : &memo[((size_t)node_table[node_of[g]] * n_profiles + p) * 256 + occ[g]];
        if (v && *v >= 0) return (uint32_t)*v;
        const uint32_t m = first_mask(row(g, p), occ[g], quirks), r = m ? score(g, m) << 8 | m : 0u;
        if (v) *v = (int32_t)r;
        return r;
    }

    // one ALLOC of profile p as isl_place_batch resolves it: the GPU and the mask, or false
    bool resolve(uint32_t p, uint32_t* gpu, uint32_t* mask) const {
        if (policy == ISL_POLICY_FIRST_FIT || policy == ISL_POLICY_RIGHT_TO_LEFT) {
            for (uint32_t k = 0; k < hi - lo; ++k) {
                const uint32_t g = policy == ISL_POLICY_RIGHT_TO_LEFT ? hi - 1 - k : lo + k;
                if (const uint32_t m = first_mask(row(g, p), occ[g], quirks)) { *gpu = g; *mask = m; return true; }
            }
            return false;
        }
        if (policy == ISL_POLICY_BEST_FIT || policy == ISL_POLICY_MIN_FRAG) {
            bool found = false;
            uint32_t best = 0;
            for (uint32_t g = lo; g < hi; ++g) {
                const uint32_t sm = scored(g, p), m = sm & 0xFFu;
                if (!m) continue;
                const uint32_t s = sm >> 8;
                if (!found || s < best) { found = true; best = s; *gpu = g; *mask = m; }
            }
            return found;
        }
        // node scoring (rules 1-5): the best node of the range, ties to the lowest; there its first admitting GPU in range
        bool found = false;
        uint32_t best = 0, best_node = 0;
        for (uint32_t v = 0; v < n_nodes; ++v) {
            const uint32_t g0 = std::max(lo, node_off[v]), g1 = std::min(hi, node_off[v + 1]);
            if (g0 >= g1) continue;
            const uint32_t t = node_table[v], w = width[t], wm = (1u << w) - 1u, cap = w * (g1 - g0);
            uint32_t busy = 0;
            bool admits = false;
            for (uint32_t g = g0; g < g1; ++g) {
                busy += (uint32_t)__builtin_popcount(occ[g] & wm);
                admits = admits || first_mask(row(g, p), occ[g], quirks);
            }
            if (!admits) continue;
            const uint32_t req = rows[(size_t)t * n_profiles + p].size;
            const uint32_t s = policy == ISL_POLICY_MOST_ALLOCATED ? 100u * (busy + req) / cap : 100u * (cap - busy - req) / cap;
            if (!found || s > best) { found = true; best = s; best_node = v; }
        }
        if (!found) return false;
        for (uint32_t g = std::max(lo, node_off[best_node]); g < std::min(hi, node_off[best_node + 1]); ++g)
            if (const uint32_t m = first_mask(row(g, p), occ[g], quirks)) { *gpu = g; *mask = m; return true; }
        return false;
    }
};

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; node_off: n_nodes + 1 offsets; node_table: the table of every node; default_size[p]: the size an unplaced
// ALLOC reports; occ: G bytes, canonical order, updated in place; [lo, hi): the canonical range.  flagged: the rules of an
// ISL_FLAG_FIRST_AVAILABLE engine (A1-A5), else those of isl_place_batch.  memo: remember the best-fit family's score of every (table,
// profile, byte).  out: n records; returns the number of PLACED records.
uint32_t fa_place(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows,
                  const uint8_t* node_table, const uint8_t* default_size, uint8_t* occ, uint32_t lo, uint32_t hi, uint32_t quirks,
                  uint32_t policy, uint32_t flagged, uint32_t n, const isl_request* in, isl_result* out, uint32_t memo) {
    Cluster c{node_off[n_nodes], n_nodes, n_profiles, quirks, policy, lo, hi, node_off, rows, node_table, occ, {}, {}, {}};
    c.node_of.resize(c.G);
    for (uint32_t v = 0; v < n_nodes; ++v)
        for (uint32_t g = node_off[v]; g < node_off[v + 1]; ++g) c.node_of[g] = v;
    c.width.assign(n_tables, 0);
    c.cand.assign(n_tables, {});
    if (memo) c.memo.assign((size_t)n_tables * n_profiles * 256, -1);
    for (uint32_t t = 0; t < n_tables; ++t)
        for (uint32_t p = 0; p < n_profiles; ++p) {
            const isl_profile& r = rows[(size_t)t * n_profiles + p];
            for (uint32_t k = 0; k < r.n_starts; ++k) {
                c.width[t] = std::max<uint32_t>(c.width[t], r.starts[k] + r.size);
                if (const uint32_t m = legal_mask(r.size, r.starts[k], quirks)) c.cand[t].push_back(m);
            }
        }
    for (uint32_t i = 0; i < n; ++i) {          // A2: every FREE first; default records for the rest
        const isl_request& r = in[i];
        if (r.op == ISL_OP_FREE) {
            const bool ok = r.handle < c.G && r.size > 0 && r.start + r.size <= 8;
            if (ok && r.handle >= lo && r.handle < hi) occ[r.handle] &= (uint8_t)~(((1u << r.size) - 1u) << r.start);
            out[i] = {r.handle, r.start, r.size, (uint16_t)(ok ? ISL_ST_FREED : ISL_ST_BAD_SPAN)};
        } else if (r.op == ISL_OP_ALLOC) {
            out[i] = r.profile < n_profiles ? isl_result{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, default_size[r.profile], (uint16_t)ISL_ST_NO_CAPACITY}
                                            : isl_result{ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_BAD_PROFILE};
        } else out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP};
    }
    uint32_t placed = 0;
    bool pod_done = false;
    for (uint32_t i = 0; i < n; ++i) {
        if (in[i].op != ISL_OP_ALLOC) continue;
        // A1: an ALLOC continues its pod when the request before it is an ALLOC with the same handle
        const bool cont = flagged && i > 0 && in[i - 1].op == ISL_OP_ALLOC && in[i - 1].handle == in[i].handle;
        if (!cont) pod_done = false;
        if (pod_done) { out[i].status = ISL_ST_ALT_SKIPPED; continue; }     // A3: the default record, status ALT_SKIPPED
        const uint32_t p = in[i].profile;
        uint32_t g, m;
        if (p >= n_profiles || !c.resolve(p, &g, &m)) continue;
        occ[g] |= (uint8_t)m;
        out[i] = {g, (uint8_t)__builtin_ctz(m), (uint8_t)__builtin_popcount(m), (uint16_t)ISL_ST_PLACED};
        pod_done = true;
        ++placed;
    }
    return placed;
}

}  // extern "C"
