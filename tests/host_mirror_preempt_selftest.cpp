// Self-test of InstasliceReconciler::PreemptPending (C++ host mirror, priority preemption) on a GPU: the known-answer vector of
// tests/golden/kat_preempt.json ("issue_table") with PriorityClass values, then the preempt -> release -> place flow for its first three
// pods.  Built and run by tests/test_gpu_preempt.py.
#include <cstdio>
#include <cstdlib>
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
    Instaslice is; is.Name = "n0"; is.Spec.Migplacement = a100_40gb();
    is.Spec.MigGPUUUID["GPU-0"] = is.Spec.MigGPUUUID["GPU-1"] = "NVIDIA A100-PCIE-40GB";
    alloc(is, "A", "GPU-0", 0, 1); alloc(is, "B", "GPU-0", 1, 1); alloc(is, "C", "GPU-0", 2, 2); alloc(is, "D", "GPU-0", 4, 1);
    alloc(is, "E", "GPU-1", 0, 4); alloc(is, "F", "GPU-1", 4, 2);
    PreparedDetails dangling; dangling.Parent = "GPU-0"; dangling.Start = 5; dangling.Size = 2;      // no pod: pinned
    is.Spec.Prepared["x"] = dangling;
    list.Items.push_back(is);
    InstasliceReconciler r;
    r.Sync(list);
    const std::map<std::string, int32_t> prio = {{"A", 100}, {"B", 100}, {"C", 200}, {"D", 500}, {"E", 200}, {"F", 100}};
    const char* profiles[] = {"1g.5gb", "2g.10gb", "3g.20gb", "1g.5gb", "1g.5gb", "4g.20gb"};
    const int32_t values[] = {300, 300, 300, 100, 200, 600};
    std::vector<PreemptPod> pods;
    for (int i = 0; i < 6; ++i) pods.push_back({Pod{"p" + std::to_string(i), "default", "p" + std::to_string(i)}, profiles[i], values[i]});
    const std::vector<PreemptOutcome> out = r.PreemptPending(list, pods, prio);
    EXPECT(out.size() == 6);
    EXPECT(out[0].verdict == PreemptVerdict::Fits && out[0].GPUUUID == "GPU-1" && out[0].Start == 6 && out[0].Size == 1);
    EXPECT(out[1].verdict == PreemptVerdict::Preempt && out[1].GPUUUID == "GPU-1" && out[1].Start == 4 && out[1].Victims == std::vector<std::string>{"F"});
    EXPECT(out[2].verdict == PreemptVerdict::Preempt && out[2].GPUUUID == "GPU-1" && out[2].Start == 0 && out[2].Size == 4 &&
           out[2].Victims == std::vector<std::string>{"E"});
    EXPECT(out[3].verdict == PreemptVerdict::None);
    EXPECT(out[4].verdict == PreemptVerdict::Preempt && out[4].GPUUUID == "GPU-0" && out[4].Start == 0 && out[4].Victims == std::vector<std::string>{"A"});
    EXPECT(out[5].verdict == PreemptVerdict::None);
    EXPECT(list.Items[0].Spec.Allocations.size() == 6);          // a query: nothing written
    FirstFitPolicy policy;
    for (int i = 0; i < 3; ++i) {                                // delete the victims, then place: each pod lands where it was told
        for (const std::string& v : out[i].Victims) EXPECT(r.Release(list, v));
        const std::vector<Outcome> placed = r.PlacePending(list, policy, {PendingPod{pods[i].pod, pods[i].ProfileName}});
        EXPECT(placed[0].verdict == Verdict::Placed);
        EXPECT(placed[0].alloc.GPUUUID == out[i].GPUUUID && placed[0].alloc.Start == out[i].Start && placed[0].alloc.Size == out[i].Size);
    }
    printf("PASS\n");
    return 0;
}
