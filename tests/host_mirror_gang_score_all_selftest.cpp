// Self-test of InstasliceReconciler::PlaceGangs (C++ host mirror) on node-scoring engines created with ISL_FLAG_GANG_NODE_SCORE |
// ISL_FLAG_GANG_NODE_SCORE_ALL, on a GPU: a few-node job's rounds go to the deepest node, then to the fuller (MostAllocated) or emptier
// (LeastAllocated) one; elastic balanced replicas are placed with their leading pods; the engine refuses the bit without
// ISL_FLAG_GANG_NODE_SCORE and keeps its other refusals.  Built and run by tests/test_gpu_gang_score_all.py.
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "../instaslice_b200/host/instaslice_host.hpp"

using namespace instaslice;

#define EXPECT(cond)                                                             \
    do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); std::exit(1); } } while (0)

static std::vector<Mig> a100_40gb() {
    struct R { const char* n; int size; std::vector<int> starts; int gi; };
    const std::vector<R> rows = {{"1g.5gb", 1, {0, 1, 2, 3, 4, 5, 6}, 0}, {"2g.10gb", 2, {0, 2, 4}, 1}, {"3g.20gb", 4, {0, 4}, 2},
                                 {"4g.20gb", 4, {0}, 3},                  {"7g.40gb", 8, {0}, 4},        {"1g.10gb", 2, {0, 2, 4, 6}, 9}};
    std::vector<Mig> out;
    for (const R& r : rows) {
        Mig m; m.Profile = r.n; m.Giprofileid = r.gi; m.CIProfileID = r.gi; m.CIEngProfileID = 0;
        for (int s : r.starts) m.Placements.push_back({r.size, s});
        out.push_back(m);
    }
    return out;
}

static Instaslice node(const std::string& name, const std::vector<std::string>& gpus) {
    Instaslice is; is.Name = name; is.Spec.Migplacement = a100_40gb();
    for (const std::string& g : gpus) is.Spec.MigGPUUUID[g] = "NVIDIA A100-PCIE-40GB";
    return is;
}

static std::vector<PendingPod> gang(const std::vector<std::string>& profiles, int& uid) {
    std::vector<PendingPod> out;
    for (const std::string& p : profiles) { out.push_back({Pod{"u" + std::to_string(uid), "default", "p" + std::to_string(uid)}, p}); ++uid; }
    return out;
}

static InstasliceList cluster() {
    InstasliceList list;
    list.Items.push_back(node("n0", {"GPU-0"})); list.Items.push_back(node("n1", {"GPU-1"}));
    return list;
}

static bool refused(uint32_t policy, uint32_t flags) {
    try { InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, policy, flags); }
    catch (const std::runtime_error&) { return true; }
    return false;
}

int main() {
    FirstFitPolicy policy;
    int uid = 0;
    const uint32_t all = ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_NODE_SCORE_ALL;
    for (uint32_t pol : {ISL_POLICY_MOST_ALLOCATED, ISL_POLICY_LEAST_ALLOCATED}) {
        const bool most = pol == ISL_POLICY_MOST_ALLOCATED;
        // three empty one-GPU nodes; a pod goes to n0 (a tie of three empty nodes); then a few-node job of nine 1g.5gb: no node takes
        // it whole, the first round goes to the deepest node, n1 (seven starts, a tie with n2 in depth and score), and the second round
        // places the last two on n0 (the fuller node, 37 against 25) under MostAllocated, on n2 (75 against 62) under LeastAllocated
        InstasliceList list = cluster();
        list.Items.push_back(node("n2", {"GPU-2"}));
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, pol,
                               all | ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_MIN_MEMBERS | ISL_FLAG_GANG_BALANCED);
        r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {gang({"1g.5gb"}, uid), gang(std::vector<std::string>(9, "1g.5gb"), uid)},
                                                          {ISL_GANG_ANY_NODES, ISL_GANG_FEW_NODES}, {0, 0});
        EXPECT(out.size() == 2 && out[0].verdict == Verdict::Placed && out[1].verdict == Verdict::Placed);
        EXPECT(out[0].allocs[0].GPUUUID == "GPU-0" && out[1].allocs.size() == 9);
        for (int k = 0; k < 7; ++k) EXPECT(out[1].allocs[k].GPUUUID == "GPU-1" && out[1].allocs[k].Start == k);
        for (int k = 7; k < 9; ++k) EXPECT(out[1].allocs[k].GPUUUID == (most ? "GPU-0" : "GPU-2"));
        r.Sync(list);                                // the CR and the engine agree
        // five 2g.10gb replicas with maxSkew 1 and a minimum of two: four find room, so the gang is placed with its first four pods
        const std::vector<GangOutcome> el = r.PlaceGangs(list, policy, {gang(std::vector<std::string>(5, "2g.10gb"), uid)},
                                                         {(uint8_t)ISL_GANG_BALANCED_NODES(1)}, {2});
        EXPECT(el.size() == 1 && el[0].verdict == Verdict::Placed && el[0].allocs.size() == 4);
        const std::vector<std::pair<std::string, int>> want =
            most ? std::vector<std::pair<std::string, int>>{{"GPU-0", 4}, {"GPU-2", 0}, {"GPU-2", 2}, {"GPU-2", 4}}
                 : std::vector<std::pair<std::string, int>>{{"GPU-0", 2}, {"GPU-2", 2}, {"GPU-0", 4}, {"GPU-2", 4}};
        for (size_t k = 0; k < want.size(); ++k) EXPECT(el[0].allocs[k].GPUUUID == want[k].first && el[0].allocs[k].Start == want[k].second);
        r.Sync(list);
    }
    EXPECT(refused(ISL_POLICY_MOST_ALLOCATED, ISL_FLAG_GANG_NODE_SCORE_ALL | ISL_FLAG_GANG_FEW_NODES));
    EXPECT(refused(ISL_POLICY_FIRST_FIT, all | ISL_FLAG_GANG_FEW_NODES));
    EXPECT(refused(ISL_POLICY_LEAST_ALLOCATED, ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_FEW_NODES));
    EXPECT(refused(ISL_POLICY_LEAST_ALLOCATED, all | ISL_FLAG_GANG_FEW_NODES | ISL_FLAG_GANG_PREEMPT));
    EXPECT(refused(ISL_POLICY_MOST_ALLOCATED, all | ISL_FLAG_GANG_BALANCED));
    EXPECT(!refused(ISL_POLICY_MOST_ALLOCATED, all | ISL_FLAG_GANG_FEW_NODES | ISL_FLAG_GANG_MIN_MEMBERS));
    EXPECT(!refused(ISL_POLICY_LEAST_ALLOCATED, all | ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_BALANCED | ISL_FLAG_GANG_MIN_MEMBERS));
    printf("host mirror gang-score-all selftest: PASS\n");
    return 0;
}
