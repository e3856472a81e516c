// ref_fast.cpp — the same allocator results from an 8-bit occupancy word per GPU.
//
// TEST INFRASTRUCTURE (see oracle.h).  PARITY UNPINNED by reference tests; pinned by
// SURVEY.md 8c known-answer vectors and by agreement with ref_faithful.cpp / ref_py.py.
//
// orc_start_for restates the search of getStartIndexFromPreparedState
// (internal/controller/instaslice_controller.go:343-383) on a bit mask; orc_fast_place restates
// the sequence  Reconcile node loop (:190) -> findDeviceForASlice GPU loop (:242) -> first hit wins
// with one monotone cursor per profile (valid because occupancy only grows between frees), i.e.
// O(R + P*G) instead of the reference's O(R * G * entries).  It is the honest strong CPU baseline
// and the verifier for the 1M-request runs.
//
// ISL_POLICY_RIGHT_TO_LEFT (the policy the reference only stubs, :464-469) is the same search over the GPUs in DESCENDING canonical
// order.  ISL_POLICY_MIN_FRAG (extension, SURVEY 8a-ext "richer score"): among the GPUs where the profile has a valid start, the one
// where taking the reference's first valid start makes the fewest (profile, start) pairs of that GPU's table infeasible, ties to the
// lowest canonical index — computed here pair by pair from the rows, independently of the engine's per-byte score table.
//
// ISL_POLICY_BEST_FIT is this repository's extension (SURVEY 8a-ext, no reference counterpart):
// among GPUs where the profile has a valid start, take the one with the fewest free slices after
// the placement (popcount over the 8-bit word), ties to the lowest canonical index; the start on
// that GPU is still the reference's first valid start.

#include "oracle.h"

#include <algorithm>
#include <vector>

extern "C" uint8_t orc_start_for(const isl_profile* row, uint32_t quirks, uint8_t occ) {
    const int needed = row->size;                                   // :334
    const bool strict = quirks & ISL_QUIRK_STRICT_BOUND;
    const bool pow2 = quirks & ISL_QUIRK_POW2_ONLY;
    uint8_t found = ISL_START_NONE;                                 // :343
    for (uint32_t k = 0; k < row->n_starts; ++k) {                  // :344 in CRD order
        const int v = row->starts[k];
        if (v >= (int)ISL_SLOTS) continue;                          // the reference would panic (Q7); tables are validated upstream
        if ((occ >> v) & 1) continue;                               // :345
        if (needed == 1) { found = (uint8_t)v; break; }             // :346-349
        const bool handled = pow2 ? (needed == 2 || needed == 4 || needed == 8) : (needed >= 2 && needed <= 8);
        if (!handled) continue;                                     // Q2
        const bool inside = strict ? (v + needed < (int)ISL_SLOTS) : (v + needed <= (int)ISL_SLOTS);   // :351,:360,:370 (Q1)
        if (!inside) continue;
        const uint32_t span = ((1u << needed) - 1u) << v;
        if (occ & span) continue;                                   // :352,:361,:371-374
        found = (uint8_t)v;
        break;                                                      // (:368-378 has no break but cannot be reached under Q1)
    }
    return found;
}

struct orc_fast {
    uint32_t G = 0, P = 0, T = 1, quirks = 0, policy = 0;
    std::vector<isl_profile> rows;     // [t*P + p]; n_starts == 0: the node's Migplacement has no row with that name
    std::vector<uint8_t> occ;
    std::vector<uint8_t> gtab;         // table of the node that owns the GPU (every node publishes its own Migplacement)
    std::vector<uint8_t> lut;          // [(t*P + p)*256 + occ] -> start or 9
    std::vector<uint32_t> cursor;      // first GPU that may still take profile p (right-to-left: one past the LAST GPU that may)
    std::vector<uint8_t> default_size; // size reported for an unplaced request: the first table that knows the name
};

extern "C" {

orc_fast* orc_fast_new_tables(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows,
                              const uint8_t* node_table, uint32_t quirks, uint32_t policy) {
    orc_fast* h = new orc_fast;
    h->G = node_off[n_nodes]; h->P = n_profiles; h->T = n_tables; h->quirks = quirks; h->policy = policy;
    h->rows.assign(rows, rows + (size_t)n_tables * n_profiles);
    h->occ.assign(h->G, 0);
    h->gtab.assign(h->G, 0);
    for (uint32_t n = 0; n < n_nodes; ++n)
        for (uint32_t g = node_off[n]; g < node_off[n + 1]; ++g) h->gtab[g] = node_table ? node_table[n] : 0;
    h->lut.resize((size_t)n_tables * n_profiles * 256);
    for (uint32_t r = 0; r < n_tables * n_profiles; ++r)
        for (uint32_t o = 0; o < 256; ++o) h->lut[(size_t)r * 256 + o] = orc_start_for(&rows[r], quirks, (uint8_t)o);
    h->cursor.assign(n_profiles, policy == ISL_POLICY_RIGHT_TO_LEFT ? h->G : 0u);
    h->default_size.assign(n_profiles, 0);
    for (uint32_t p = 0; p < n_profiles; ++p)       // first node in canonical order whose Migplacement has the name
        for (uint32_t n = 0; n < n_nodes; ++n) {
            const isl_profile& r = rows[(size_t)(node_table ? node_table[n] : 0) * n_profiles + p];
            if (r.n_starts) { h->default_size[p] = r.size; break; }
        }
    return h;
}
orc_fast* orc_fast_new(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_profiles, const isl_profile* rows,
                       uint32_t quirks, uint32_t policy) {
    return orc_fast_new_tables(n_nodes, node_off, 1, n_profiles, rows, nullptr, quirks, policy);
}
void orc_fast_delete(orc_fast* h) { delete h; }
void orc_fast_load(orc_fast* h, const uint8_t* occ) {
    std::copy(occ, occ + h->G, h->occ.begin());
    std::fill(h->cursor.begin(), h->cursor.end(), h->policy == ISL_POLICY_RIGHT_TO_LEFT ? h->G : 0u);
}
void orc_fast_occupancy(orc_fast* h, uint8_t* out) { std::copy(h->occ.begin(), h->occ.end(), out); }

int orc_fast_place(orc_fast* h, uint32_t n, const isl_request* in, isl_result* out) {
    for (uint32_t i = 0; i < n; ++i) {                              // canonical batch: FREEs first
        if (in[i].op == ISL_OP_ALLOC) continue;
        if (in[i].op != ISL_OP_FREE) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP}; continue; }   // NOOP and any unknown op
        const uint32_t g = in[i].handle, st = in[i].start, sz = in[i].size;
        if (g >= h->G || sz == 0 || st + sz > ISL_SLOTS) { out[i] = {g, (uint8_t)st, (uint8_t)sz, (uint16_t)ISL_ST_BAD_SPAN}; continue; }
        h->occ[g] &= (uint8_t)~(((1u << sz) - 1u) << st);
        for (uint32_t p = 0; p < h->P; ++p) h->cursor[p] = h->policy == ISL_POLICY_RIGHT_TO_LEFT ? std::max(h->cursor[p], g + 1) : std::min(h->cursor[p], g);
        out[i] = {g, (uint8_t)st, (uint8_t)sz, (uint16_t)ISL_ST_FREED};
    }
    for (uint32_t i = 0; i < n; ++i) {                              // then ALLOCs in request order
        if (in[i].op != ISL_OP_ALLOC) continue;
        const uint32_t p = in[i].profile;
        if (p >= h->P) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_BAD_PROFILE}; continue; }
        // the start table and the size are those of the node that owns the GPU (each node's own Migplacement, :332-340)
        auto lut_of = [&](uint32_t g) { return &h->lut[((size_t)h->gtab[g] * h->P + p) * 256]; };
        uint32_t hit = ISL_GPU_NONE;
        if (h->policy == ISL_POLICY_FIRST_FIT) {
            uint32_t g = h->cursor[p];
            while (g < h->G && lut_of(g)[h->occ[g]] == ISL_START_NONE) ++g;
            h->cursor[p] = g;
            if (g < h->G) hit = g;
        } else if (h->policy == ISL_POLICY_RIGHT_TO_LEFT) {
            uint32_t g = h->cursor[p];                               // one past the last GPU that may still take p
            while (g > 0 && lut_of(g - 1)[h->occ[g - 1]] == ISL_START_NONE) --g;
            h->cursor[p] = g;
            if (g > 0) hit = g - 1;
        } else if (h->policy == ISL_POLICY_MIN_FRAG) {
            int best = 1 << 30;
            for (uint32_t g = 0; g < h->G; ++g) {
                const uint8_t s = lut_of(g)[h->occ[g]];
                if (s == ISL_START_NONE) continue;
                const isl_profile* trows = &h->rows[(size_t)h->gtab[g] * h->P];
                const uint8_t before = h->occ[g], after = (uint8_t)(before | (((1u << trows[p].size) - 1u) << s));
                int lost = 0;                                         // (profile, start) pairs feasible before and not after
                for (uint32_t q = 0; q < h->P; ++q)
                    for (uint32_t k = 0; k < trows[q].n_starts; ++k) {
                        isl_profile one = trows[q];
                        one.n_starts = 1; one.starts[0] = trows[q].starts[k];
                        const bool was = orc_start_for(&one, h->quirks, before) != ISL_START_NONE;
                        const bool is = orc_start_for(&one, h->quirks, after) != ISL_START_NONE;
                        lost += was && !is;
                    }
                if (lost < best) { best = lost; hit = g; }
            }
        } else {
            int best = 1 << 30;
            for (uint32_t g = 0; g < h->G; ++g) {
                const uint8_t s = lut_of(g)[h->occ[g]];
                if (s == ISL_START_NONE) continue;
                const uint8_t sz = h->rows[(size_t)h->gtab[g] * h->P + p].size;
                const uint8_t after = (uint8_t)(h->occ[g] | (((1u << sz) - 1u) << s));
                const int free_after = 8 - __builtin_popcount(after);
                if (free_after < best) { best = free_after; hit = g; }
            }
        }
        if (hit == ISL_GPU_NONE) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, h->default_size[p], (uint16_t)ISL_ST_NO_CAPACITY}; continue; }
        const uint8_t s = lut_of(hit)[h->occ[hit]];
        const uint8_t size = h->rows[(size_t)h->gtab[hit] * h->P + p].size;
        h->occ[hit] |= (uint8_t)(((1u << size) - 1u) << s);
        out[i] = {hit, s, size, (uint16_t)ISL_ST_PLACED};
    }
    return ISL_OK;
}

}  // extern "C"
