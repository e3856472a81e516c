// bestfit_fast.cpp — brute-force restatement of k_bestfit (isl_place_batch on ISL_POLICY_BEST_FIT / _MIN_FRAG engines, and isl_place_gangs
// on an engine without a gang flag, every policy) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_bestfit.  Every FREE of the call is applied first (inside [lo, hi) only); then, gang
// after gang, each ALLOC member scans every GPU of [lo, hi) in scan order (right-to-left: from the top) and takes the one with the lowest
// score, the first in scan order on a tie.  A gang whose member finds nothing is undone byte by byte.  A batch is a call of gangs of one.
// It keeps no class structure, no minimum and no score table of the engine: it shares nothing with the kernel but the rules.
#include <cstdint>
#include <utility>
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
    std::vector<int32_t> memo;              // [table][profile][byte]: score << 8 | mask, -1 until first asked; empty: no memo
};

// score << 8 | mask of profile p on byte o of a GPU of table t: mask = its first legal start (0: none); score = what the policy minimises
// (best-fit: free slices after; min-frag: (profile, start) pairs of the table that stop being feasible, counted pair by pair; first-fit
// family: 0)
int32_t evaluate(const Ctx& c, uint32_t t, uint32_t p, uint32_t o) {
    const isl_profile* trows = c.rows + (size_t)t * c.n_profiles;
    const uint32_t mine = first_mask(trows[p], o, c.quirks);
    if (!mine) return 0;
    uint32_t s = 0;
    if (c.policy == ISL_POLICY_BEST_FIT) s = 8u - (uint32_t)__builtin_popcount(o | mine);
    else if (c.policy == ISL_POLICY_MIN_FRAG)
        for (uint32_t q = 0; q < c.n_profiles; ++q)
            for (uint32_t k = 0; k < trows[q].n_starts; ++k) {
                const uint32_t m = legal_mask(trows[q].size, trows[q].starts[k], c.quirks);
                s += m && !(o & m) && ((o | mine) & m);
            }
    return (int32_t)(s << 8 | mine);
}

// evaluate(); with the memo on, each (table, profile, byte) is walked once, the first time a GPU asks for it
int32_t lookup(Ctx& c, uint32_t t, uint32_t p, uint32_t o) {
    if (c.memo.empty()) return evaluate(c, t, p, o);
    int32_t& v = c.memo[((size_t)t * c.n_profiles + p) * 256 + o];
    if (v < 0) v = evaluate(c, t, p, o);
    return v;
}

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; gtab: the table of every GPU (G bytes, canonical order); occ: G bytes (canonical), updated in place;
// default_size[p]: the size an unplaced ALLOC reports; [lo, hi): the canonical range; memo: remember every evaluation per (table, profile,
// byte); gang_off: n_gangs + 1 offsets (a batch: gangs of one).  out as isl_place_gangs / isl_place_batch_range write it.
void bff_place_gangs(uint32_t G, uint32_t n_profiles, const isl_profile* rows, const uint8_t* gtab, const uint8_t* default_size, uint8_t* occ,
                     uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy, uint32_t n_gangs, const uint32_t* gang_off,
                     const isl_request* in, isl_result* out, uint32_t memo) {
    Ctx c{n_profiles, quirks, policy, rows, {}};
    if (memo) {
        uint32_t n_tables = 1;
        for (uint32_t g = 0; g < G; ++g) n_tables = gtab[g] + 1u > n_tables ? gtab[g] + 1u : n_tables;
        c.memo.assign((size_t)n_tables * n_profiles * 256, -1);
    }
    const uint32_t n = gang_off[n_gangs];
    const bool descending = policy == ISL_POLICY_RIGHT_TO_LEFT;
    const bool first_hit = policy == ISL_POLICY_FIRST_FIT || descending;     // every score is 0: the first admitting GPU wins
    for (uint32_t i = 0; i < n; ++i) {                  // FREEs first; default records for the rest
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
    std::vector<std::pair<uint32_t, uint8_t>> undo;     // (GPU, byte before) of the open gang's placements
    for (uint32_t gi = 0; gi < n_gangs; ++gi) {
        undo.clear();
        uint32_t failed = n;
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1] && failed == n; ++i) {
            if (in[i].op != ISL_OP_ALLOC) continue;
            const uint32_t p = in[i].profile;
            if (p >= n_profiles) { failed = i; break; }
            bool found = false;
            uint32_t best_g = 0;
            int32_t best = 0;
            for (uint32_t k = 0; k < hi - lo; ++k) {
                const uint32_t g = descending ? hi - 1 - k : lo + k;
                const int32_t v = lookup(c, gtab[g], p, occ[g]);
                if (!(v & 0xFF)) continue;
                if (!found || (v >> 8) < (best >> 8)) { found = true; best_g = g; best = v; }
                if (first_hit) break;
            }
            if (!found) { failed = i; break; }
            const uint32_t mine = (uint32_t)best & 0xFFu;
            undo.push_back({best_g, occ[best_g]});
            occ[best_g] |= (uint8_t)mine;
            out[i] = {best_g, (uint8_t)__builtin_ctz(mine), (uint8_t)__builtin_popcount(mine), (uint16_t)ISL_ST_PLACED};
        }
        if (failed == n) continue;
        for (size_t k = undo.size(); k-- > 0;) occ[undo[k].first] = undo[k].second;
        for (uint32_t i = gang_off[gi]; i < gang_off[gi + 1]; ++i) {     // rule 4: every other ALLOC member is GANG_ABORTED
            if (in[i].op != ISL_OP_ALLOC || i == failed) continue;
            const uint32_t p = in[i].profile;
            out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)(p < n_profiles ? default_size[p] : 0), (uint16_t)ISL_ST_GANG_ABORTED};
        }
    }
}

}  // extern "C"
