// Self-test of InstasliceReconciler::PlaceGangs (C++ host mirror, all-or-nothing pod groups) on a GPU: the hand-derived
// known-answer vector of include/islplace.h's gang rules, a gang across two nodes, and the Prepared veto (:198-203) releasing a
// whole gang.  Built and run by tests/test_gpu_gangs.py.
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

int main() {
    FirstFitPolicy policy;
    int uid = 0;
    {   // one empty GPU, reference-exact quirks: the five gangs of the known-answer vector in one call
        InstasliceList list; list.Items.push_back(node("n0", {"GPU-0"}));
        InstasliceReconciler r; r.Sync(list);
        const std::vector<std::vector<PendingPod>> gangs = {gang({"3g.20gb", "3g.20gb"}, uid), gang({"3g.20gb", "1g.5gb"}, uid),
                                                            gang({"1g.5gb", "2g.10gb"}, uid), gang({"1g.5gb", "1g.5gb"}, uid), gang({"1g.5gb"}, uid)};
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, gangs);
        EXPECT(out.size() == 5);
        EXPECT(out[0].verdict == Verdict::None && out[0].allocs.empty());
        EXPECT(out[1].verdict == Verdict::Placed && out[1].allocs.size() == 2 && out[1].allocs[0].Start == 0 && out[1].allocs[0].Size == 4 &&
               out[1].allocs[1].Start == 4 && out[1].allocs[1].Size == 1 && out[1].allocs[1].PodUUID == gangs[1][1].pod.UID);
        EXPECT(out[2].verdict == Verdict::None);
        EXPECT(out[3].verdict == Verdict::Placed && out[3].allocs[0].Start == 5 && out[3].allocs[1].Start == 6);
        EXPECT(out[4].verdict == Verdict::None);
        EXPECT(InstasliceReconciler::occupancyByte(list.Items[0], "GPU-0") == 0x7F);
        EXPECT(list.Items[0].Spec.Allocations.size() == 4);      // placed gangs only
        r.Sync(list);                                             // the CR and the engine agree: nothing of an aborted gang is left
        EXPECT(r.PlaceGangs(list, policy, {gang({"1g.5gb"}, uid)})[0].verdict == Verdict::None);
    }
    {   // a gang may span GPUs and nodes
        InstasliceList list; list.Items.push_back(node("n0", {"GPU-0"})); list.Items.push_back(node("n1", {"GPU-1"}));
        InstasliceReconciler r; r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {gang({"3g.20gb", "3g.20gb"}, uid)});
        EXPECT(out[0].verdict == Verdict::Placed && out[0].allocs[0].GPUUUID == "GPU-0" && out[0].allocs[1].GPUUUID == "GPU-1");
        EXPECT(out[0].allocs[0].Nodename == "n0" && out[0].allocs[1].Nodename == "n1");
    }
    {   // the exact-match Prepared veto on one member releases the whole gang; the next gang sees none of it
        InstasliceList list; list.Items.push_back(node("n0", {"GPU-0"}));
        PreparedDetails p; p.Profile = "1g.5gb"; p.Start = 1; p.Size = 1; p.Parent = "GPU-0"; p.PodUUID = "gone";
        list.Items[0].Spec.Prepared["MIG-x"] = p;
        InstasliceReconciler r; r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {gang({"1g.5gb", "1g.5gb"}, uid), gang({"2g.10gb", "1g.5gb"}, uid)});
        EXPECT(out[0].verdict == Verdict::Veto && out[0].allocs.empty());
        EXPECT(out[1].verdict == Verdict::Placed && out[1].allocs[0].Start == 0 && out[1].allocs[1].Start == 2);
        EXPECT(list.Items[0].Spec.Allocations.size() == 2);
    }
    printf("host mirror gangs selftest: PASS\n");
    return 0;
}
