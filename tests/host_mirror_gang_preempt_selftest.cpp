// Self-test of InstasliceReconciler::PreemptPendingGangs (C++ host mirror, gang preemption) on a GPU: the one-node vector of
// tests/golden/kat_gang_preempt.json ("one_node_two_cheap_victims") with PriorityClass values, under ISL_FLAG_GANG_PREEMPT |
// ISL_FLAG_GANG_ONE_NODE and the reference-free quirk set, then the preempt -> release -> place flow for that gang, and the refusal of a
// gang whose pods carry two priorities.  Built and run by tests/test_gpu_gang_preempt.py.
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

static void alloc(Instaslice& is, const std::string& uid, const std::string& gpu, uint32_t start, uint32_t size) {
    AllocationDetails a; a.PodUUID = uid; a.GPUUUID = gpu; a.Start = start; a.Size = size; a.Allocationstatus = "created";
    is.Spec.Allocations[uid] = a;
}

int main() {
    InstasliceList list;
    for (int n = 0; n < 2; ++n) {
        Instaslice is; is.Name = "n" + std::to_string(n); is.Spec.Migplacement = a100_40gb();
        is.Spec.MigGPUUUID["GPU-" + std::to_string(n)] = "NVIDIA A100-PCIE-40GB";
        list.Items.push_back(is);
    }
    alloc(list.Items[0], "big", "GPU-0", 0, 8);                 // node 0: one 7g victim of value 300
    alloc(list.Items[1], "s1", "GPU-1", 0, 4);                  // node 1: two 3g victims of values 100 and 200
    alloc(list.Items[1], "s2", "GPU-1", 4, 4);
    InstasliceReconciler r(ISL_QUIRKS_FIXED, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_PREEMPT | ISL_FLAG_GANG_ONE_NODE);
    r.Sync(list);
    const std::map<std::string, int32_t> prio = {{"big", 300}, {"s1", 100}, {"s2", 200}};
    std::vector<PreemptPod> gang;
    for (int i = 0; i < 2; ++i) gang.push_back({Pod{"w" + std::to_string(i), "default", "w" + std::to_string(i)}, "3g.20gb", 500});
    const std::vector<GangPreemptOutcome> out = r.PreemptPendingGangs(list, {gang}, prio);
    EXPECT(out.size() == 1 && out[0].verdict == PreemptVerdict::Preempt);
    EXPECT((out[0].Victims == std::vector<std::string>{"s1", "s2"}));      // (3, 3, 2) on node 1 beats (4, 3, 1) on node 0
    EXPECT(out[0].pods.size() == 2 && out[0].pods[0].GPUUUID == "GPU-1" && out[0].pods[0].Start == 0 && out[0].pods[1].Start == 4);
    EXPECT(list.Items[1].Spec.Allocations.size() == 2);          // a query: nothing written
    for (const std::string& v : out[0].Victims) EXPECT(r.Release(list, v));
    FirstFitPolicy policy;
    std::vector<PendingPod> pending;
    for (const PreemptPod& p : gang) pending.push_back(PendingPod{p.pod, p.ProfileName});
    const std::vector<GangOutcome> placed = r.PlaceGangs(list, policy, {pending});
    EXPECT(placed[0].verdict == Verdict::Placed && placed[0].allocs.size() == 2);
    for (int i = 0; i < 2; ++i)
        EXPECT(placed[0].allocs[i].GPUUUID == "GPU-1" && placed[0].allocs[i].Start == out[0].pods[i].Start);
    gang[1].Priority = 400;
    bool threw = false;
    try { r.PreemptPendingGangs(list, {gang}, prio); } catch (const std::runtime_error&) { threw = true; }
    EXPECT(threw);
    printf("PASS\n");
    return 0;
}
