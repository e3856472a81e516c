// preempt_fast.cpp — brute-force restatement of isl_preempt (include/islplace.h, rules 1-6) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of the device kernels and the single-core CPU baseline of tools/preempt_time.py.  For
// every preemptor it scores every (GPU, start of the row) pair of the range with the five keys of rule 5 as a tuple, then applies the
// winner: V's spans are released, the preemptor's span becomes busy and pinned.  It shares nothing with the kernels but the rules.
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <tuple>
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

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; gtab: table of every GPU; occ: G bytes (canonical order); [lo, hi): the canonical range searched.
// Returns ISL_OK or ISL_EINVAL (rule 2, rule 3's FREE); out / evict as isl_preempt writes them.
int pf_preempt(uint32_t G, uint32_t n_profiles, const isl_profile* rows, const uint8_t* gtab, const uint8_t* default_size,
               const uint8_t* occ_in, uint32_t lo, uint32_t hi, uint32_t quirks, uint32_t policy, uint32_t n, const isl_request* in,
               const uint8_t* priority, uint32_t n_victims, const isl_victim* victims, isl_result* out, uint32_t* evict) {
    std::vector<uint8_t> occ(occ_in, occ_in + G);
    std::vector<uint32_t> owner((size_t)G * 8, ISL_GPU_NONE);       // victim index of every slice, NONE = free or pinned
    for (uint32_t i = 0; i < n; ++i) if (in[i].op == ISL_OP_FREE) return ISL_EINVAL;
    for (uint32_t k = 0; k < n_victims; ++k) {
        const isl_victim& v = victims[k];
        if (v.gpu >= G || v.size == 0 || v.start + v.size > 8) return ISL_EINVAL;
        if (v.gpu < lo || v.gpu >= hi) continue;
        for (uint32_t s = v.start; s < (uint32_t)v.start + v.size; ++s) {
            if (!((occ[v.gpu] >> s) & 1u) || owner[(size_t)v.gpu * 8 + s] != ISL_GPU_NONE) return ISL_EINVAL;
            owner[(size_t)v.gpu * 8 + s] = k;
        }
    }
    const bool descending = policy == ISL_POLICY_RIGHT_TO_LEFT;
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t* row_out = evict + (size_t)i * 8;
        for (uint32_t j = 0; j < 8; ++j) row_out[j] = ISL_GPU_NONE;
        if (in[i].op != ISL_OP_ALLOC) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP}; continue; }
        const uint32_t p = in[i].profile, pi = priority[i];
        if (p >= n_profiles) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_BAD_PROFILE}; continue; }
        using Key = std::tuple<uint32_t, uint32_t, uint32_t, uint32_t, uint32_t>;
        bool found = false;
        Key best{};
        uint32_t best_g = 0, best_m = 0;
        std::vector<uint32_t> best_v;
        for (uint32_t pos = 0; pos < hi - lo; ++pos) {
            const uint32_t g = descending ? hi - 1 - pos : lo + pos;
            const isl_profile& row = rows[(size_t)gtab[g] * n_profiles + p];
            for (uint32_t k = 0; k < row.n_starts; ++k) {
                const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
                if (!m) continue;
                uint32_t V[8], nV = 0;
                bool ok = true;
                for (uint32_t s = 0; s < 8 && ok; ++s) {
                    if (!((m >> s) & 1u) || !((occ[g] >> s) & 1u)) continue;
                    const uint32_t v = owner[(size_t)g * 8 + s];
                    if (v == ISL_GPU_NONE || victims[v].priority >= pi) { ok = false; break; }
                    bool seen = false;
                    for (uint32_t x = 0; x < nV; ++x) seen |= V[x] == v;
                    if (!seen) V[nV++] = v;
                }
                if (!ok) continue;
                uint32_t mx = 0, sum = 0;
                for (uint32_t x = 0; x < nV; ++x) { mx = std::max<uint32_t>(mx, victims[V[x]].priority + 1u); sum += victims[V[x]].priority; }
                const Key key{mx, sum, nV, pos, k};
                if (!found || key < best) { found = true; best = key; best_g = g; best_m = m; best_v.assign(V, V + nV); }
            }
        }
        if (!found) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, default_size[p], (uint16_t)ISL_ST_NO_CAPACITY}; continue; }
        std::sort(best_v.begin(), best_v.end());
        for (size_t j = 0; j < best_v.size(); ++j) {
            const isl_victim& v = victims[best_v[j]];
            row_out[j] = best_v[j];
            for (uint32_t s = v.start; s < (uint32_t)v.start + v.size; ++s) owner[(size_t)best_g * 8 + s] = ISL_GPU_NONE;
            occ[best_g] &= (uint8_t)~(((1u << v.size) - 1u) << v.start);
        }
        occ[best_g] |= (uint8_t)best_m;               // busy and pinned: no victim owns these slices
        for (uint32_t s = 0; s < 8; ++s) if ((best_m >> s) & 1u) owner[(size_t)best_g * 8 + s] = ISL_GPU_NONE;
        out[i] = {best_g, (uint8_t)__builtin_ctz(best_m), (uint8_t)__builtin_popcount(best_m), (uint16_t)ISL_ST_PLACED};
    }
    return ISL_OK;
}

}  // extern "C"
