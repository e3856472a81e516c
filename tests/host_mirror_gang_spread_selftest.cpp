// Self-test of InstasliceReconciler::PlaceGangs (C++ host mirror) on an engine created with ISL_FLAG_GANG_DISTINCT_NODES, on a GPU: a gang
// that an unflagged engine puts on one GPU lands on three nodes, a gang with more members than nodes is committed nowhere, and the engine
// refuses the flag together with ISL_FLAG_GANG_ONE_NODE.  Built and run by tests/test_gpu_gang_spread.py.
#include <cstdio>
#include <cstdlib>
#include <set>
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
    list.Items.push_back(node("n0", {"GPU-0", "GPU-1"})); list.Items.push_back(node("n1", {"GPU-2"})); list.Items.push_back(node("n2", {"GPU-3"}));
    return list;
}

int main() {
    FirstFitPolicy policy;
    int uid = 0;
    {   // three replicas land on three nodes; four replicas on three nodes abort and leave nothing behind
        InstasliceList list = cluster();
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_DISTINCT_NODES);
        r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {gang({"1g.5gb", "1g.5gb", "1g.5gb"}, uid),
                                                                         gang({"1g.5gb", "1g.5gb", "1g.5gb", "1g.5gb"}, uid)});
        EXPECT(out.size() == 2);
        EXPECT(out[0].verdict == Verdict::Placed && out[0].allocs.size() == 3);
        EXPECT(out[0].allocs[0].GPUUUID == "GPU-0" && out[0].allocs[1].GPUUUID == "GPU-2" && out[0].allocs[2].GPUUUID == "GPU-3");
        std::set<std::string> nodes;
        for (const AllocationDetails& a : out[0].allocs) nodes.insert(a.Nodename);
        EXPECT(nodes.size() == 3);
        EXPECT(out[1].verdict == Verdict::None && out[1].allocs.empty());
        EXPECT(list.Items[0].Spec.Allocations.size() == 1 && list.Items[1].Spec.Allocations.size() == 1 && list.Items[2].Spec.Allocations.size() == 1);
        r.Sync(list);                                             // the CR and the engine agree
        const std::vector<GangOutcome> again = r.PlaceGangs(list, policy, {gang({"1g.5gb", "1g.5gb"}, uid)});
        EXPECT(again[0].verdict == Verdict::Placed && again[0].allocs[0].GPUUUID == "GPU-0" && again[0].allocs[0].Start == 1 &&
               again[0].allocs[1].GPUUUID == "GPU-2" && again[0].allocs[1].Start == 1);
    }
    {   // an unflagged engine puts the same three replicas on one GPU
        InstasliceList list = cluster();
        InstasliceReconciler r; r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {gang({"1g.5gb", "1g.5gb", "1g.5gb"}, uid)});
        EXPECT(out[0].verdict == Verdict::Placed);
        for (const AllocationDetails& a : out[0].allocs) EXPECT(a.GPUUUID == "GPU-0");
    }
    bool refused = false;
    try { InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_DISTINCT_NODES | ISL_FLAG_GANG_ONE_NODE); }
    catch (const std::runtime_error&) { refused = true; }
    EXPECT(refused);
    printf("host mirror gang-spread selftest: PASS\n");
    return 0;
}
