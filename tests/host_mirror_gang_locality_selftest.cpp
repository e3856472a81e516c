// Self-test of InstasliceReconciler::PlaceGangs with one locality per gang (C++ host mirror) on an engine created with
// ISL_FLAG_GANG_LOCALITY, on a GPU: a one-node gang, a distinct-node gang, an any-node gang and a gang with no room go through one call
// on one occupancy; a locality list of the wrong length throws, and the engine refuses the flag with ISL_FLAG_GANG_FEW_NODES.  Built and
// run by tests/test_gpu_gang_locality.py.
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

int main() {
    FirstFitPolicy policy;
    int uid = 0;
    {   // nodes of one, one and two GPUs (reference-exact quirks: 3g.20gb only at slice 0)
        InstasliceList list;
        list.Items.push_back(node("n0", {"GPU-0"})); list.Items.push_back(node("n1", {"GPU-1"})); list.Items.push_back(node("n2", {"GPU-2", "GPU-3"}));
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_LOCALITY);
        r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(
            list, policy, {gang({"3g.20gb", "3g.20gb"}, uid), gang({"1g.5gb", "1g.5gb"}, uid), gang({"1g.5gb", "1g.5gb"}, uid), gang({"7g.40gb"}, uid)},
            {ISL_GANG_ONE_NODE, ISL_GANG_DISTINCT_NODES, ISL_GANG_ANY_NODES, ISL_GANG_ANY_NODES});
        EXPECT(out.size() == 4);
        // only node 2 takes both 3g.20gb
        EXPECT(out[0].verdict == Verdict::Placed && out[0].allocs[0].Nodename == "n2" && out[0].allocs[1].Nodename == "n2");
        // one 1g.5gb per node: the first on GPU-0, the second on the next node
        EXPECT(out[1].verdict == Verdict::Placed && out[1].allocs[0].GPUUUID == "GPU-0" && out[1].allocs[1].GPUUUID == "GPU-1");
        // anywhere: both on the first admitting GPU, GPU-0, after the distinct-node gang's slice
        EXPECT(out[2].verdict == Verdict::Placed && out[2].allocs[0].GPUUUID == "GPU-0" && out[2].allocs[1].GPUUUID == "GPU-0");
        EXPECT(out[2].allocs[0].Start == 1 && out[2].allocs[1].Start == 2);
        EXPECT(out[3].verdict == Verdict::None && out[3].allocs.empty());     // no GPU is empty
        EXPECT(list.Items[0].Spec.Allocations.size() == 3 && list.Items[1].Spec.Allocations.size() == 1 && list.Items[2].Spec.Allocations.size() == 2);
        r.Sync(list);                                             // the CR and the engine agree
        EXPECT(r.PlaceGangs(list, policy, {gang({"1g.5gb", "1g.5gb"}, uid)}, {ISL_GANG_FEW_NODES})[0].verdict == Verdict::Placed);
        bool threw = false;
        try { r.PlaceGangs(list, policy, {gang({"1g.5gb"}, uid)}, {ISL_GANG_ONE_NODE, ISL_GANG_ONE_NODE}); }
        catch (const std::runtime_error&) { threw = true; }
        EXPECT(threw);
    }
    bool refused = false;
    try { InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_FEW_NODES); }
    catch (const std::runtime_error&) { refused = true; }
    EXPECT(refused);
    printf("host mirror gang-locality selftest: PASS\n");
    return 0;
}
