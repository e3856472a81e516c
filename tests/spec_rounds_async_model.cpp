// spec_rounds_async_model.cpp — the speculative rounds under ARBITRARY interleavings of the stages (test infrastructure).
//
// spec_rounds_model.cpp steps all stages in lock step.  On the device they are not: a stage goes on as soon as the records it needs are
// there, a stage in front may be rounds ahead, a certified stage stops publishing rounds and its FINAL record stands for every round from
// the one it was certified in, the exit heads live in two slots per stage (round parity) guarded by an ack word of the reader.  This model
// runs the same protocol with a random scheduler that picks, step by step, any stage that can proceed, and checks soundness (a certified
// entry is the true token), freedom from deadlock, termination — and that a reader never needs a record that has been overwritten.
//
// Record words are self-validating: a reader takes any word whose tag (24 bits of the call's tag, and the round) matches.  Two more
// modes model what the record memory may hold when a call starts (argument 3):
//   1  the records of an EARLIER call on other requests, over the same stages, carry this call's tag (stream ids s and s + 2^24 of a
//      partitioned inventory, whose shared record memory is never cleared between calls): the device would take them as current
//   2  this call's tag is 0 and the memory is cleared: only the round-0 mass words (tag 0, round 0) match a cleared word, so a stage may
//      read 0 for the masses of stages in front that have not published yet; rounds >= 1 and final words never match a cleared word
#define SPEC_MODEL_NO_MAIN
#include "spec_rounds_model.cpp"

struct DRec { bool valid = false; long dq = 0, dr = 0; bool c = false; };
struct XSlot { int round = 0; Heads x; bool cur = false; };      // cur: written by this call
struct Final { bool valid = false; int rf = 0; Heads x; long dq = 0, dr = 0; };
// fault injection (the tests check that the model notices): 1 = a final record stands for EVERY round, 2 = no flow control of the exit
// slots, 3 = a final record is preferred over the round's own record
static int fault = 0;
static int stale = 0;
// the records a call leaves behind (what a stale-tag call of mode 1 finds)
static struct { uint32_t S = 0; std::vector<std::vector<DRec>> dhist; std::vector<XSlot> xslot; std::vector<Final> fin; } left;

static int run_async(uint32_t G, uint32_t seg, uint32_t n_req, int table, bool bounded, uint32_t fill_mask, int bias) {
    World w;
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
    const uint32_t S = (G + seg - 1) / seg;
    std::vector<Heads> truth(S + 1, Heads(np, 0));
    for (uint32_t s = 0; s < S; ++s) { truth[s + 1] = truth[s]; uint64_t d; simulate(w, s * seg, std::min(G, (s + 1) * seg), truth[s + 1], ~0ull, &d); }
    std::vector<int> big, small;
    for (int p = 0; p < np; ++p) { if (w.prof[p].masks.empty() || w.q[p].empty()) continue; (w.prof[p].size >= 4 ? big : small).push_back(p); }
    auto massq = [&](const Heads& h) { long m = 0; for (int p : big) m += h[p]; return m; };
    auto massr = [&](const Heads& h) { long m = 0; for (int p : small) m += (long)h[p] * w.prof[p].size; return m; };
    std::vector<long> Q(S), Rw(S), Ro(S);
    uint32_t us = 0; for (int p : small) for (uint32_t m : w.prof[p].masks) us |= m;
    for (uint32_t s = 0; s < S; ++s) for (uint32_t g = s * seg; g < std::min(G, (s + 1) * seg); ++g) {
        uint32_t o = w.occ[g];
        for (int it = 0; it < 2; ++it) { uint32_t best = 0; for (int p : big) for (uint32_t m : w.prof[p].masks) if (!(o & m) && __builtin_popcount(m) > __builtin_popcount(best)) best = m; if (!best) break; o |= best; ++Q[s]; }
        Rw[s] += __builtin_popcount(~o & us); Ro[s] += __builtin_popcount(~(uint32_t)w.occ[g] & us);
    }
    long totb = 0, tots = 0; for (int p : big) totb += w.q[p].size(); for (int p : small) tots += (long)w.q[p].size() * w.prof[p].size;
    const int RMAX = (int)S + 8;
    std::vector<Heads> H(S, Heads(np, 0)), X(S, Heads(np, 0)), Hc(S, Heads(np, 0)), Xc(S, Heads(np, 0)), predA(S, Heads(np, 0)), predB(S, Heads(np, 0));
    for (uint32_t s = 1; s < S; ++s) {      // round 0: the masses of the stages in front (mode 2: each read as 0 by a reader that came early)
        long qs = 0, rs = 0;
        for (uint32_t j = 0; j < s; ++j) { const bool zero = stale == 2 && rnd() % 2; if (!zero) { rs += qs < totb ? Rw[j] : Ro[j]; qs += Q[j]; } }
        spread(w, H[s], big, std::min(qs, totb), false); spread(w, H[s], small, std::min(rs, tots), true);
    }
    std::vector<char> done(S, 0), cprev(S, 0), logvalid(S, 0), have(S, 0), known(S, 0), need(S, 1), phase(S, 0), havepred(S, 0);
    std::vector<int> round(S, 1);
    std::vector<uint64_t> maxdec(S, 0);
    std::vector<long> Dq(S, 0), Dr(S, 0);
    std::vector<std::vector<DRec>> dhist(RMAX + 1, std::vector<DRec>(S));
    std::vector<XSlot> xslot(2 * S);
    std::vector<int> ack(S, 0);
    std::vector<Final> fin(S);
    if (stale == 1 && left.S == S) {
        dhist = left.dhist; xslot = left.xslot; fin = left.fin;
        for (auto& x : xslot) x.cur = false;
    }
    cprev[0] = 1; known[0] = 1;
    uint32_t n_done = 0;
    uint64_t steps = 0;
    while (n_done < S) {
        if (++steps > 400ull * S * RMAX) { printf("FAIL: livelock\n"); return 1; }
        // a random stage that is not done; blocked stages are skipped; all blocked = deadlock
        // bias 0: any stage; 1: the stage furthest in front that can move (stages in front run as far ahead as the flow control lets them);
        // 2: the stage furthest behind that can move; 3: mostly one of them, now and then any
        const int b = bias == 3 ? (rnd() % 4 == 0 ? 0 : 1 + (int)(rnd() % 2)) : bias;
        uint32_t start = b == 0 ? (uint32_t)(rnd() % S) : 0u;
        bool progressed = false;
        for (uint32_t k = 0; k < S && !progressed; ++k) {
            const uint32_t s = b == 2 ? S - 1 - k : (start + k) % S;
            if (done[s]) continue;
            const int r = round[s];
            if (r > RMAX) { printf("FAIL: stage %u beyond %d rounds\n", s, RMAX); return 1; }
            if (phase[s] == 0) {
                // flow control of the two exit slots: the successor must have read round r - 2
                if (fault != 2 && r >= 3 && s + 1 < S && !(ack[s + 1] + 2 >= r)) continue;
                if (need[s]) {
                    Heads h = H[s]; uint64_t d;
                    const uint64_t cap = bounded && have[s] && !known[s] ? (maxdec[s] * 21 >> 4) + 8 : ~0ull;
                    const bool complete = simulate(w, s * seg, std::min(G, (s + 1) * seg), h, cap, &d);
                    if (complete) { X[s] = h; Hc[s] = H[s]; Xc[s] = h; have[s] = 1; logvalid[s] = 1; maxdec[s] = std::max(maxdec[s], d); }
                    else { Heads e = Xc[s]; spread(w, e, big, massq(H[s]) - massq(Hc[s]), false); spread(w, e, small, massr(H[s]) - massr(Hc[s]), true);
                           for (int p = 0; p < np; ++p) e[p] = std::max(e[p], H[s][p]); X[s] = e; logvalid[s] = 0; }
                    Dq[s] = massq(X[s]) - massq(H[s]); Dr[s] = massr(X[s]) - massr(H[s]);
                }
                // overwriting a slot the successor has not read would lose a record it still needs
                if (s + 1 < S && xslot[2 * s + (r & 1)].cur && !done[s + 1] && ack[s + 1] < xslot[2 * s + (r & 1)].round) { printf("FAIL: exit slot overwritten before it was read\n"); return 1; }
                xslot[2 * s + (r & 1)] = XSlot{r, X[s], true};
                dhist[r][s] = DRec{true, Dq[s], Dr[s], (bool)cprev[s]};
                phase[s] = 1; progressed = true;
            } else {
                // gather: this round's records of every stage in front (the round's own record first; a final record stands for every round
                // from the one its stage was certified in), the exit of the stage right in front
                bool ready = true, allc = true, allc_bp = true; long sq = 0, sr = 0;
                for (uint32_t j = 0; j < s && ready; ++j) {
                    bool c; long dq, dr;
                    if (dhist[r][j].valid && fault != 3) { c = dhist[r][j].c; dq = dhist[r][j].dq; dr = dhist[r][j].dr; }
                    else if (fin[j].valid && (fin[j].rf <= r || fault == 1)) { c = true; dq = fin[j].dq; dr = fin[j].dr; }
                    else { ready = false; break; }
                    allc_bp = allc; allc = allc && c; sq += dq; sr += dr;
                }
                Heads xp(np, 0);
                if (ready && s > 0) {
                    if (xslot[2 * (s - 1) + (r & 1)].round == r) xp = xslot[2 * (s - 1) + (r & 1)].x;
                    else if (fin[s - 1].valid && fin[s - 1].rf <= r) xp = fin[s - 1].x;
                    else if (xslot[2 * (s - 1) + (r & 1)].round > r && xslot[2 * (s - 1) + (r & 1)].cur) { printf("FAIL: the exit of round %d was overwritten by round %d before stage %u read it\n", r, xslot[2 * (s - 1) + (r & 1)].round, s); return 1; }
                    else ready = false;
                }
                if (!ready) continue;
                ack[s] = r;
                if (allc && cprev[s]) {
                    if (!logvalid[s]) { printf("FAIL: certified with a cut-off log\n"); return 1; }
                    if (H[s] != truth[s] || X[s] != truth[s + 1]) { printf("FAIL: unsound certification at stage %u round %d\n", s, r); return 1; }
                    fin[s] = Final{true, r, X[s], Dq[s], Dr[s]};
                    ack[s] = 0xFFFF; done[s] = 1; ++n_done; progressed = true;
                    continue;
                }
                const bool cnow = s == 0 ? true : (H[s] == xp);
                Heads h = xp;
                if (s > 0) {
                    spread(w, h, big, sq - massq(h), false); spread(w, h, small, sr - massr(h), true);
                    long ea = 0, eb = 0;
                    if (havepred[s]) for (int p = 0; p < np; ++p) { ea += std::labs((long)predA[s][p] - (long)xp[p]); eb += std::labs((long)predB[s][p] - (long)xp[p]); }
                    predA[s] = h; predB[s] = xp; havepred[s] = 1;
                    if (eb < ea) h = xp;
                    if (allc && cnow && h != H[s]) { printf("FAIL: the correction moved a consistent entry\n"); return 1; }
                } else h = H[s];
                known[s] = allc_bp;
                need[s] = h != H[s] || !logvalid[s];
                cprev[s] = cnow && logvalid[s];
                H[s] = h;
                round[s] = r + 1; phase[s] = 0; progressed = true;
            }
        }
        if (!progressed) { printf("FAIL: deadlock (%u of %u stages done)\n", n_done, S); return 1; }
    }
    left.S = S; left.dhist = dhist; left.xslot = xslot; left.fin = fin;
    return 0;
}

int main(int argc, char** argv) {
    const int cases = argc > 1 ? atoi(argv[1]) : 60;
    fault = argc > 2 ? atoi(argv[2]) : 0;
    const int mode = argc > 3 ? atoi(argv[3]) : 0;
    int bad = 0;
    for (int i = 0; i < cases && !bad; ++i) {
        const uint32_t seg = 16u << (rnd() % 4);
        const uint32_t S = 2 + (uint32_t)(rnd() % 40);
        const uint32_t G = seg * S - (uint32_t)(rnd() % seg);
        const uint32_t n_req = 1 + (uint32_t)(rnd() % (6 * G));
        const uint32_t fills[] = {0x00, 0x7F, 0xFF, 0x15, 0x33};
        const int tbl = (int)(rnd() % 3); const uint32_t fm = fills[rnd() % 5];
        if (mode == 1) {        // an earlier call on other requests over the same stages, then this one
            stale = 0;
            const uint32_t n0 = 1 + (uint32_t)(rnd() % (6 * G));
            if (run_async(G, seg, n0, tbl, i % 2 == 1, fills[rnd() % 5], i % 4)) { printf("FAIL: the earlier call\n"); return 1; }
        }
        stale = mode;
        bad |= run_async(G, seg, n_req, tbl, i % 2 == 1, fm, i % 4);
        if (bad) printf("case %d: G %u seg %u requests %u table %d bounded %d fill %#x\n", i, G, seg, n_req, tbl, i % 2, fm);
    }
    printf(bad ? "spec rounds async model: FAILED\n" : "spec rounds async model: ok (%d cases)\n", cases);
    return bad;
}
