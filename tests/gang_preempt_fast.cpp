// gang_preempt_fast.cpp — brute-force restatement of isl_preempt on an ISL_FLAG_GANG_PREEMPT engine (include/islplace.h, rules 1-6 and
// P1-P8) on flat occupancy bytes.
//
// TEST INFRASTRUCTURE: the large-scale checker of k_preempt_gangs and the single-core CPU baseline of tools/gang_preempt_time.py.  Every
// member is chosen by scoring every (GPU, start of the row) pair it may use with the five keys of rule 5 as a tuple; a one-node gang is
// tried on every node and undone, then replayed on the node of least (max + 1, sum, count, scan position).  It shares nothing with the
// kernels but the rules.
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

using Key = std::tuple<uint32_t, uint32_t, uint32_t, uint32_t, uint32_t>;

struct Undo {
    uint32_t g;
    uint8_t occ;
    uint32_t owner[8];
};

struct World {
    uint32_t n_profiles, lo, hi, quirks;
    bool descending;
    const isl_profile* rows;
    const uint8_t* gtab;
    const isl_victim* victims;
    std::vector<uint8_t> occ;
    std::vector<uint32_t> owner;       // victim index of every slice, NONE = free or pinned
    std::vector<Undo> log;

    struct Pick {
        bool found = false;
        Key key{};
        uint32_t g = 0, m = 0;
        std::vector<uint32_t> V;
    };

    // rules 4-5 for one preemptor over the scan positions [p0, p1) whose GPU `ok` admits
    template <typename Ok>
    Pick pick(uint32_t p, uint32_t pi, uint32_t p0, uint32_t p1, Ok ok) const {
        Pick best;
        for (uint32_t pos = p0; pos < p1; ++pos) {
            const uint32_t g = descending ? hi - 1 - pos : lo + pos;
            if (!ok(g)) continue;
            const isl_profile& row = rows[(size_t)gtab[g] * n_profiles + p];
            for (uint32_t k = 0; k < row.n_starts; ++k) {
                const uint32_t m = legal_mask(row.size, row.starts[k], quirks);
                if (!m) continue;
                uint32_t V[8], nV = 0;
                bool good = true;
                for (uint32_t s = 0; s < 8 && good; ++s) {
                    if (!((m >> s) & 1u) || !((occ[g] >> s) & 1u)) continue;
                    const uint32_t v = owner[(size_t)g * 8 + s];
                    if (v == ISL_GPU_NONE || victims[v].priority >= pi) { good = false; break; }
                    bool seen = false;
                    for (uint32_t x = 0; x < nV; ++x) seen |= V[x] == v;
                    if (!seen) V[nV++] = v;
                }
                if (!good) continue;
                uint32_t mx = 0, sum = 0;
                for (uint32_t x = 0; x < nV; ++x) { mx = std::max<uint32_t>(mx, victims[V[x]].priority + 1u); sum += victims[V[x]].priority; }
                const Key key{mx, sum, nV, pos, k};
                if (!best.found || key < best.key) { best.found = true; best.key = key; best.g = g; best.m = m; best.V.assign(V, V + nV); }
            }
        }
        std::sort(best.V.begin(), best.V.end());
        return best;
    }

    // the victims of `c` leave, its span becomes busy and pinned; the GPU's prior state goes to the log
    void apply(const Pick& c) {
        Undo u{c.g, occ[c.g], {}};
        std::memcpy(u.owner, &owner[(size_t)c.g * 8], sizeof u.owner);
        log.push_back(u);
        for (uint32_t v : c.V) {
            const isl_victim& x = victims[v];
            for (uint32_t s = x.start; s < (uint32_t)x.start + x.size; ++s) owner[(size_t)c.g * 8 + s] = ISL_GPU_NONE;
            occ[c.g] &= (uint8_t)~(((1u << x.size) - 1u) << x.start);
        }
        occ[c.g] |= (uint8_t)c.m;
        for (uint32_t s = 0; s < 8; ++s) if ((c.m >> s) & 1u) owner[(size_t)c.g * 8 + s] = ISL_GPU_NONE;
    }

    void undo_to(size_t mark) {
        while (log.size() > mark) {
            const Undo& u = log.back();
            occ[u.g] = u.occ;
            std::memcpy(&owner[(size_t)u.g * 8], u.owner, sizeof u.owner);
            log.pop_back();
        }
    }
};

isl_result unplaced(uint32_t size, uint32_t status) { return {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, (uint8_t)size, (uint16_t)status}; }

}  // namespace

extern "C" {

// rows[t * n_profiles + p]; gtab: table of every GPU; occ: G bytes (canonical order); node_off: n_nodes + 1 canonical offsets; [lo, hi):
// the canonical partition.  locality: ISL_GANG_ANY_NODES, _ONE_NODE or _DISTINCT_NODES for every gang, or 4 for each gang's `start`
// byte (ISL_FLAG_GANG_LOCALITY).  Returns ISL_OK or ISL_EINVAL (rule 2, rule 3's FREE, P1); out / evict as isl_preempt writes them.
int gpf_preempt(uint32_t G, uint32_t n_profiles, const isl_profile* rows, const uint8_t* gtab, const uint8_t* default_size,
                const uint8_t* occ_in, uint32_t n_nodes, const uint32_t* node_off, uint32_t lo, uint32_t hi, uint32_t quirks,
                uint32_t policy, uint32_t locality, uint32_t n, const isl_request* in, const uint8_t* priority, uint32_t n_victims,
                const isl_victim* victims, isl_result* out, uint32_t* evict) {
    World w{n_profiles, lo, hi, quirks, policy == ISL_POLICY_RIGHT_TO_LEFT, rows, gtab, victims, {occ_in, occ_in + G},
            std::vector<uint32_t>((size_t)G * 8, ISL_GPU_NONE), {}};
    for (uint32_t i = 0; i < n; ++i) if (in[i].op == ISL_OP_FREE) return ISL_EINVAL;
    std::vector<uint32_t> goff;                                 // P1: maximal runs of equal handles, each with its locality
    std::vector<uint8_t> gloc;
    for (uint32_t i = 0; i < n; ++i) if (i == 0 || in[i].handle != in[i - 1].handle) goff.push_back(i);
    goff.push_back(n);
    for (size_t g = 0; g + 1 < goff.size(); ++g) {
        int prio = -1, loc = -1;
        for (uint32_t r = goff[g]; r < goff[g + 1]; ++r) {
            if (in[r].op != ISL_OP_ALLOC) continue;
            if (prio >= 0 && priority[r] != prio) return ISL_EINVAL;
            prio = priority[r];
            if (locality == 4) {
                const int b = in[r].start;
                if (b == 2 || b > 3 || (loc >= 0 && b != loc)) return ISL_EINVAL;
                loc = b;
            }
        }
        gloc.push_back(locality == 4 ? (uint8_t)std::max(loc, 0) : (uint8_t)locality);
    }
    for (uint32_t k = 0; k < n_victims; ++k) {
        const isl_victim& v = victims[k];
        if (v.gpu >= G || v.size == 0 || v.start + v.size > 8) return ISL_EINVAL;
        if (v.gpu < lo || v.gpu >= hi) continue;
        for (uint32_t s = v.start; s < (uint32_t)v.start + v.size; ++s) {
            if (!((w.occ[v.gpu] >> s) & 1u) || w.owner[(size_t)v.gpu * 8 + s] != ISL_GPU_NONE) return ISL_EINVAL;
            w.owner[(size_t)v.gpu * 8 + s] = k;
        }
    }
    auto node_of = [&](uint32_t g) { return (uint32_t)(std::upper_bound(node_off, node_off + n_nodes + 1, g) - node_off) - 1; };
    for (uint32_t i = 0; i < n; ++i) {                          // defaults
        for (uint32_t j = 0; j < 8; ++j) evict[(size_t)i * 8 + j] = ISL_GPU_NONE;
        out[i] = in[i].op != ISL_OP_ALLOC ? unplaced(0, ISL_ST_NOOP)
                 : in[i].profile >= n_profiles ? unplaced(0, ISL_ST_BAD_PROFILE)
                                               : unplaced(default_size[in[i].profile], ISL_ST_NO_CAPACITY);
    }
    auto abort_others = [&](uint32_t r0, uint32_t r1, uint32_t keep_rank) {
        uint32_t rank = 0;
        for (uint32_t r = r0; r < r1; ++r) {
            if (in[r].op != ISL_OP_ALLOC) continue;
            if (rank++ == keep_rank) continue;
            out[r] = unplaced(in[r].profile < n_profiles ? default_size[in[r].profile] : 0u, ISL_ST_GANG_ABORTED);
            for (uint32_t j = 0; j < 8; ++j) evict[(size_t)r * 8 + j] = ISL_GPU_NONE;
        }
    };
    auto place = [&](uint32_t r, const World::Pick& c) {
        out[r] = {c.g, (uint8_t)__builtin_ctz(c.m), (uint8_t)__builtin_popcount(c.m), (uint16_t)ISL_ST_PLACED};
        for (size_t j = 0; j < c.V.size(); ++j) evict[(size_t)r * 8 + j] = c.V[j];
    };
    const uint32_t Gr = hi - lo;
    for (size_t gi = 0; gi + 1 < goff.size(); ++gi) {
        const uint32_t r0 = goff[gi], r1 = goff[gi + 1];
        w.log.clear();
        if (gloc[gi] != ISL_GANG_ONE_NODE) {                   // P3 any node / distinct nodes, P5 rule 4
            std::vector<uint32_t> used;
            uint32_t rank = 0;
            bool failed = false;
            for (uint32_t r = r0; r < r1 && !failed; ++r) {
                if (in[r].op != ISL_OP_ALLOC) continue;
                World::Pick c;
                if (in[r].profile < n_profiles)
                    c = w.pick(in[r].profile, priority[r], 0, Gr, [&](uint32_t g) {
                        return gloc[gi] != ISL_GANG_DISTINCT_NODES || std::find(used.begin(), used.end(), node_of(g)) == used.end();
                    });
                if (!c.found) {
                    w.undo_to(0);
                    abort_others(r0, r1, rank);
                    failed = true;
                    break;
                }
                w.apply(c);
                place(r, c);
                used.push_back(node_of(c.g));
                ++rank;
            }
            continue;
        }
        // P3 one node: every node of the partition in scan order, tried on the state and undone
        const uint32_t j_lo = node_of(lo), j_hi = node_of(hi - 1) + 1;
        bool any = false;
        std::tuple<uint32_t, uint32_t, uint32_t, uint32_t> best{};
        uint32_t best_j = 0, D = 0;
        for (uint32_t jj = 0; jj < j_hi - j_lo; ++jj) {
            const uint32_t j = w.descending ? j_hi - 1 - jj : j_lo + jj;
            const uint32_t a = std::max(node_off[j], lo), b = std::min(node_off[j + 1], hi);
            if (a >= b) continue;
            const uint32_t p0 = w.descending ? hi - b : a - lo, p1 = w.descending ? hi - a : b - lo;
            uint32_t depth = 0, mx = 0, sum = 0, cnt = 0;
            bool all = true;
            for (uint32_t r = r0; r < r1; ++r) {
                if (in[r].op != ISL_OP_ALLOC) continue;
                World::Pick c;
                if (in[r].profile < n_profiles) c = w.pick(in[r].profile, priority[r], p0, p1, [](uint32_t) { return true; });
                if (!c.found) { all = false; break; }
                mx = std::max(mx, std::get<0>(c.key)); sum += std::get<1>(c.key); cnt += std::get<2>(c.key);
                w.apply(c);
                ++depth;
            }
            w.undo_to(0);
            D = std::max(D, depth);
            const auto key = std::make_tuple(mx, sum, cnt, jj);
            if (all && (!any || key < best)) { any = true; best = key; best_j = j; }
        }
        if (!any) { abort_others(r0, r1, D); continue; }
        const uint32_t a = std::max(node_off[best_j], lo), b = std::min(node_off[best_j + 1], hi);
        const uint32_t p0 = w.descending ? hi - b : a - lo, p1 = w.descending ? hi - a : b - lo;
        for (uint32_t r = r0; r < r1; ++r) {
            if (in[r].op != ISL_OP_ALLOC) continue;
            const World::Pick c = w.pick(in[r].profile, priority[r], p0, p1, [](uint32_t) { return true; });
            w.apply(c);
            place(r, c);
        }
    }
    return ISL_OK;
}

}  // extern "C"
