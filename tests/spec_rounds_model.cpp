// spec_rounds_model.cpp — CPU model of the speculative rounds of k_pipeline (DESIGN.md 4.5), test infrastructure.
//
// The device protocol, restated sequentially: stages = contiguous GPU ranges; every stage simulates its range with the exact GPU-major
// first-fit recurrence from a PREDICTED entry (queue heads), publishes its exit heads X and the group masses it consumed D, corrects its
// entry from X of the stage in front and the mass sums of all stages in front, and is certified when the consistency bits c(j, r-1) of all
// j <= s are set.  This model checks, on random inventories / request mixes / tables, the properties the kernel relies on:
//   soundness     a stage is never certified with an entry that is not the true token (checked against the sequential recurrence)
//   progress      every round certifies at least one more stage; rounds <= stages + 1
//   no-op         a consistent prefix is not moved by the correction (so "certified" implies "the log in shared memory is the log")
//   bounded sims  cutting a simulation off and extrapolating its exit never certifies a cut-off log
// It shares no code with the kernel: prediction, correction and certification are re-derived here from the design.
// Random mode: spec_rounds_model [cases].  Given workload: spec_rounds_model --world FILE [--bounded] (tests/spec_workloads.py writes it)
// prints the rounds until the last stage was certified and the stage count.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static uint64_t rnd() { uint64_t z = (rng_state += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }

struct Profile { int size; std::vector<uint32_t> masks; };
typedef std::vector<uint32_t> Heads;

struct World {
    std::vector<Profile> prof;
    std::vector<uint8_t> occ;
    std::vector<std::vector<uint32_t>> q;      // per profile: request times, ascending
};

// the exact recurrence over GPUs [lo, hi) from entry heads h; at most `cap` decisions (returns false when cut off)
static bool simulate(const World& w, uint32_t lo, uint32_t hi, Heads& h, uint64_t cap, uint64_t* dec) {
    const int np = (int)w.prof.size();
    uint64_t d = 0;
    for (uint32_t g = lo; g < hi; ++g) {
        uint32_t o = w.occ[g];
        while (true) {
            uint32_t best = 0xFFFFFFFFu, bm = 0; int bp = -1;
            for (int p = 0; p < np; ++p) {
                if (h[p] >= w.q[p].size()) continue;
                uint32_t m = 0;
                for (uint32_t mm : w.prof[p].masks) if ((o & mm) == 0) { m = mm; break; }
                if (!m) continue;
                if (w.q[p][h[p]] < best) { best = w.q[p][h[p]]; bp = p; bm = m; }
            }
            if (bp < 0) break;
            if (d >= cap) { *dec = d; return false; }
            o |= bm; ++h[bp]; ++d;
        }
    }
    *dec = d;
    return true;
}

// move the heads of `grp` so that their mass changes by d: shares proportional to the queue lengths, the last single-slice member (a
// group without one: its last member) takes the remainder
static void spread(const World& w, Heads& h, const std::vector<int>& grp, long d, bool weighted) {
    if (d == 0 || grp.empty()) return;
    double tot = 0;
    for (int p : grp) tot += (double)w.q[p].size() * (weighted ? w.prof[p].size : 1);
    int last = -1;
    for (int p : grp) if (!weighted || w.prof[p].size <= 1) last = p;
    if (last < 0) last = grp.back();
    long used = 0;
    std::vector<long> dp(w.prof.size(), 0);
    for (int p : grp) if (p != last) { dp[p] = tot > 0 ? std::lround((double)d * w.q[p].size() / tot) : 0; used += dp[p] * (weighted ? w.prof[p].size : 1); }
    dp[last] = (d - used) / (weighted ? w.prof[last].size : 1);
    for (int p : grp) { long v = (long)h[p] + dp[p]; h[p] = (uint32_t)std::max(0l, std::min<long>(v, (long)w.q[p].size())); }
}

// random inventory, request mix and table (the random mode below)
static World random_world(uint32_t G, uint32_t n_req, int table, uint32_t fill_mask) {
    World w;
    // tables: (size, starts) under the reference's quirks (strict bound) or the repaired rule
    auto add = [&](int size, std::vector<int> starts, bool strict) {
        Profile p; p.size = size;
        for (int v : starts) { if (size > 1 && (strict ? !(v + size < 8) : !(v + size <= 8))) continue; p.masks.push_back((((1u << size) - 1u) << v) & 0xFFu); }
        w.prof.push_back(p);
    };
    if (table == 0) { add(1, {0, 1, 2, 3, 4, 5, 6}, true); add(2, {0, 2, 4, 6}, true); add(4, {0, 4}, true); add(4, {0}, true); add(8, {0}, true); }
    else if (table == 1) { add(1, {0, 1, 2, 3, 4, 5, 6}, false); add(2, {0, 2, 4}, false); add(4, {0, 4}, false); add(4, {0}, false); add(8, {0}, false); }
    else { add(1, {0, 1, 2, 3}, true); add(2, {0, 2}, true); add(4, {0}, true); add(1, {4, 5, 6}, true); }
    const int np = (int)w.prof.size();
    w.occ.resize(G);
    for (auto& o : w.occ) o = (uint8_t)(rnd() & rnd() & fill_mask);
    w.q.assign(np, {});
    for (uint32_t t = 0; t < n_req; ++t) { int p = (int)(rnd() % (np + 1)); if (p < np && !w.prof[p].masks.empty()) w.q[p].push_back(t); }
    return w;
}

// The round loop over one world, GPUs [0, G) in stages of seg GPUs.  Returns 0 (and the rounds until the last stage was certified in
// *rounds_out) or 1 after a FAIL: line.
static int run_world(const World& w, uint32_t G, uint32_t seg, bool bounded, int* rounds_out) {
    const int np = (int)w.prof.size();
    const uint32_t S = (G + seg - 1) / seg;
    // truth
    std::vector<Heads> truth(S + 1, Heads(np, 0));
    for (uint32_t s = 0; s < S; ++s) { truth[s + 1] = truth[s]; uint64_t d; simulate(w, s * seg, std::min(G, (s + 1) * seg), truth[s + 1], ~0ull, &d); }
    // groups
    std::vector<int> big, small;
    for (int p = 0; p < np; ++p) { if (w.prof[p].masks.empty() || w.q[p].empty()) continue; (w.prof[p].size >= 4 ? big : small).push_back(p); }
    auto massq = [&](const Heads& h) { long m = 0; for (int p : big) m += h[p]; return m; };
    auto massr = [&](const Heads& h) { long m = 0; for (int p : small) m += (long)h[p] * w.prof[p].size; return m; };
    // round 0: masses per stage from the occupancy, predicted entries
    std::vector<long> Q(S), Rw(S), Ro(S);
    uint32_t us = 0; for (int p : small) for (uint32_t m : w.prof[p].masks) us |= m;
    for (uint32_t s = 0; s < S; ++s) for (uint32_t g = s * seg; g < std::min(G, (s + 1) * seg); ++g) {
        uint32_t o = w.occ[g];
        for (int it = 0; it < 2; ++it) { uint32_t best = 0; for (int p : big) for (uint32_t m : w.prof[p].masks) if (!(o & m) && __builtin_popcount(m) > __builtin_popcount(best)) best = m; if (!best) break; o |= best; ++Q[s]; }
        Rw[s] += __builtin_popcount(~o & us); Ro[s] += __builtin_popcount(~(uint32_t)w.occ[g] & us);
    }
    long totb = 0, tots = 0; for (int p : big) totb += w.q[p].size(); for (int p : small) tots += (long)w.q[p].size() * w.prof[p].size;
    std::vector<Heads> H(S, Heads(np, 0)), X(S, Heads(np, 0)), Hc(S, Heads(np, 0)), Xc(S, Heads(np, 0));
    { long qs = 0, rs = 0; for (uint32_t s = 0; s < S; ++s) { if (s) { spread(w, H[s], big, std::min(qs, totb), false); spread(w, H[s], small, std::min(rs, tots), true); } rs += qs < totb ? Rw[s] : Ro[s]; qs += Q[s]; } }
    std::vector<bool> certified(S, false), cprev(S, false), logvalid(S, false), have(S, false), known(S, false), need(S, true);
    std::vector<uint64_t> maxdec(S, 0);
    std::vector<Heads> predA(S, Heads(np, 0)), predB(S, Heads(np, 0)); std::vector<bool> havepred(S, false);
    std::vector<long> Dq(S, 0), Dr(S, 0);
    cprev[0] = true; known[0] = true;
    uint32_t n_cert = 0;
    int round = 1;
    for (; n_cert < S; ++round) {
        if (getenv("SPEC_MODEL_VERBOSE")) { uint32_t f = 0; while (f < S && certified[f]) ++f; uint32_t e = 0; while (e < S && H[e] == truth[e]) ++e; printf("round %d: certified prefix %u, exact entries prefix %u of %u\n", round, f, e, S); }
        if (round > (int)S + 2) { printf("FAIL: no termination (G %u seg %u)\n", G, seg); return 1; }
        // simulate
        for (uint32_t s = 0; s < S; ++s) {
            if (certified[s] || !need[s]) continue;
            Heads h = H[s]; uint64_t d;
            const uint64_t cap = bounded && have[s] && !known[s] ? (maxdec[s] * 21 >> 4) + 8 : ~0ull;
            const bool complete = simulate(w, s * seg, std::min(G, (s + 1) * seg), h, cap, &d);
            if (complete) { X[s] = h; Hc[s] = H[s]; Xc[s] = h; have[s] = true; logvalid[s] = true; maxdec[s] = std::max(maxdec[s], d); }
            else {      // extrapolated exit; the log is unusable
                Heads e = Xc[s];
                spread(w, e, big, massq(H[s]) - massq(Hc[s]), false); spread(w, e, small, massr(H[s]) - massr(Hc[s]), true);
                for (int p = 0; p < np; ++p) e[p] = std::max(e[p], H[s][p]);
                X[s] = e; logvalid[s] = false;
            }
            Dq[s] = massq(X[s]) - massq(H[s]); Dr[s] = massr(X[s]) - massr(H[s]);
        }
        // exchange (all stages read the same round's records; certified stages' records stand)
        std::vector<bool> cnew(S, false), newly(S, false);
        std::vector<Heads> Hn = H;
        bool allc = true, allc_before_pred = true; long sq = 0, sr = 0;        // allc_before_pred: the same over all stages in front EXCEPT the one right in front
        uint32_t newcert = 0;
        for (uint32_t s = 0; s < S; ++s) {
            // allc here = every stage in front published a set c bit (a certified stage counts as set)
            if (!certified[s]) {
                if (allc && cprev[s]) {
                    if (!logvalid[s]) { printf("FAIL: certified with a cut-off log\n"); return 1; }
                    if (H[s] != truth[s] || X[s] != truth[s + 1]) { printf("FAIL: unsound certification at stage %u round %d\n", s, round); return 1; }
                    newly[s] = true; ++newcert;
                } else {
                    cnew[s] = s == 0 ? true : (H[s] == X[s - 1]);
                    if (s > 0) {
                        Heads h = X[s - 1];
                        spread(w, h, big, sq - massq(h), false); spread(w, h, small, sr - massr(h), true);
                        {   // two candidates, the Newton step and plain chaining: the rule whose candidate of the previous round came closer to X(s-1) now
                            long ea = 0, eb = 0;
                            if (havepred[s]) for (int p = 0; p < np; ++p) { ea += std::labs((long)predA[s][p] - (long)X[s - 1][p]); eb += std::labs((long)predB[s][p] - (long)X[s - 1][p]); }
                            predA[s] = h; predB[s] = X[s - 1]; havepred[s] = true;
                            if (eb < ea) h = X[s - 1];
                        }
                        if (allc && cnew[s] && h != H[s]) { printf("FAIL: the correction moved a consistent entry\n"); return 1; }
                        Hn[s] = h;
                    }
                    // The stage whose entry becomes the true one in the NEXT round is the one behind a consistent prefix whose last member's bit
                    // is not set yet (that member's entry became the true one only this round): knowledge lags a round, so a stage is exempt from
                    // the cut-off as soon as everything but the stage right in front of it is consistent.
                    known[s] = getenv("SPEC_MODEL_STRICT_KNOWN") ? allc : allc_before_pred;
                }
            }
            allc_before_pred = allc;
            allc = allc && (certified[s] || cprev[s]);
            sq += Dq[s]; sr += Dr[s];
        }
        if (newcert == 0 && round > 1) {
            // progress: the first uncertified stage must have had the true entry this round and becomes certified next round at the latest
            uint32_t f = 0; while (f < S && certified[f]) ++f;
            if (f < S && Hn[f] != truth[f]) { printf("FAIL: no progress at stage %u round %d\n", f, round); return 1; }
        }
        for (uint32_t s = 0; s < S; ++s) {
            if (newly[s]) { certified[s] = true; ++n_cert; continue; }
            if (certified[s]) continue;
            need[s] = Hn[s] != H[s] || !logvalid[s];
            cprev[s] = cnew[s] && logvalid[s];
            H[s] = Hn[s];
        }
    }
    if (rounds_out) *rounds_out = round - 1;
    return 0;
}

static int run_case(uint32_t G, uint32_t seg, uint32_t n_req, int table, bool bounded, uint32_t fill_mask) {
    const World w = random_world(G, n_req, table, fill_mask);
    return run_world(w, G, seg, bounded, nullptr);
}

// A given workload, as whitespace-separated numbers:
//   G seg n_profiles
//   per profile: size n_masks mask...            (the masks in the order the start search tries them)
//   G occupancy bytes
//   per profile: n_requests time...              (ascending request times)
static bool read_world(const char* path, World& w, uint32_t& G, uint32_t& seg) {
    FILE* f = fopen(path, "r");
    if (!f) return false;
    bool ok = true;
    auto num = [&]() -> uint64_t { unsigned long long v = 0; if (fscanf(f, "%llu", &v) != 1) ok = false; return (uint64_t)v; };
    G = (uint32_t)num(); seg = (uint32_t)num();
    const uint32_t np = (uint32_t)num();
    for (uint32_t p = 0; p < np && ok; ++p) {
        Profile pr; pr.size = (int)num();
        const uint32_t nm = (uint32_t)num();
        for (uint32_t k = 0; k < nm && ok; ++k) pr.masks.push_back((uint32_t)num());
        w.prof.push_back(pr);
    }
    w.occ.resize(G);
    for (uint32_t g = 0; g < G && ok; ++g) w.occ[g] = (uint8_t)num();
    w.q.assign(np, {});
    for (uint32_t p = 0; p < np && ok; ++p) {
        const uint32_t n = (uint32_t)num();
        for (uint32_t i = 0; i < n && ok; ++i) w.q[p].push_back((uint32_t)num());
        for (uint32_t i = 1; i < n && ok; ++i) ok = w.q[p][i - 1] < w.q[p][i];
    }
    fclose(f);
    return ok && G > 0 && seg > 0;
}

#ifndef SPEC_MODEL_NO_MAIN
int main(int argc, char** argv) {
    if (argc > 2 && std::string(argv[1]) == "--world") {       // spec_rounds_model --world FILE [--bounded]
        World w; uint32_t G = 0, seg = 0;
        if (!read_world(argv[2], w, G, seg)) { printf("FAIL: cannot read world %s\n", argv[2]); return 2; }
        const bool bounded = argc > 3 && std::string(argv[3]) == "--bounded";
        int rounds = 0;
        const int bad = run_world(w, G, seg, bounded, &rounds);
        if (!bad) printf("rounds %d stages %u\n", rounds, (G + seg - 1) / seg);
        return bad;
    }
    const int cases = argc > 1 ? atoi(argv[1]) : 60;
    int bad = 0;
    for (int i = 0; i < cases && !bad; ++i) {
        const uint32_t seg = 16u << (rnd() % 4);                            // 16 .. 128 GPUs per stage
        const uint32_t S = 2 + (uint32_t)(rnd() % 40);
        const uint32_t G = seg * S - (uint32_t)(rnd() % seg);
        const uint32_t n_req = 1 + (uint32_t)(rnd() % (6 * G));
        const uint32_t fills[] = {0x00, 0x7F, 0xFF, 0x15, 0x33};
        const int tbl = (int)(rnd() % 3); const uint32_t fm = fills[rnd() % 5];
        if (getenv("SPEC_MODEL_CASE") && atoi(getenv("SPEC_MODEL_CASE")) != i) continue;
        bad |= run_case(G, seg, n_req, tbl, i % 2 == 1, fm);
        if (bad) printf("case %d: G %u seg %u requests %u table %d bounded %d fill %#x\n", i, G, seg, n_req, tbl, i % 2, fm);
    }
    printf(bad ? "spec rounds model: FAILED\n" : "spec rounds model: ok (%d cases)\n", cases);
    return bad;
}
#endif
