// Self-test of InstasliceReconciler::PlaceGangs with one minimum per gang (C++ host mirror) on an engine created with
// ISL_FLAG_GANG_MIN_MEMBERS, on a GPU: a gang whose leading pods reach its minimum is placed with those pods only and only their
// allocations are written, a gang below its minimum is not placed, the minimum goes with a locality per gang, a minimum list of the wrong
// length throws, and the engine refuses the flag with ISL_FLAG_ALL_NODES.  Built and run by tests/test_gpu_gang_min.py.
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
    {   // three one-GPU nodes (reference-exact quirks: 4g.20gb only at slice 0, so one per GPU)
        InstasliceList list;
        list.Items.push_back(node("n0", {"GPU-0"})); list.Items.push_back(node("n1", {"GPU-1"})); list.Items.push_back(node("n2", {"GPU-2"}));
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_MIN_MEMBERS);
        r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(
            list, policy, {gang({"4g.20gb", "4g.20gb", "4g.20gb", "4g.20gb"}, uid), gang({"1g.5gb", "1g.5gb"}, uid), gang({"4g.20gb"}, uid)},
            {}, {2, 0, 0});
        EXPECT(out.size() == 3);
        // the first three pods fit, one per GPU, and reach the minimum 2: the gang is placed without its fourth pod
        EXPECT(out[0].verdict == Verdict::Placed && out[0].allocs.size() == 3);
        EXPECT(out[0].allocs[0].GPUUUID == "GPU-0" && out[0].allocs[1].GPUUUID == "GPU-1" && out[0].allocs[2].GPUUUID == "GPU-2");
        EXPECT(out[1].verdict == Verdict::Placed && out[1].allocs.size() == 2 && out[1].allocs[0].Start == 4 && out[1].allocs[1].Start == 5);
        EXPECT(out[2].verdict == Verdict::None && out[2].allocs.empty());
        EXPECT(list.Items[0].Spec.Allocations.size() == 3 && list.Items[1].Spec.Allocations.size() == 1 && list.Items[2].Spec.Allocations.size() == 1);
        EXPECT(list.Items[0].Spec.Allocations.count("u3") == 0 && list.Items[1].Spec.Allocations.count("u3") == 0 &&
               list.Items[2].Spec.Allocations.count("u3") == 0);     // the trimmed pod has no allocation
        r.Sync(list);                                             // the CR and the engine agree
        // seven 1g.5gb fit (slice 6 of GPU-0, slices 4-6 of GPU-1 and GPU-2): a gang of eight with m = 0 needs all eight and is not placed
        const std::vector<GangOutcome> more = r.PlaceGangs(list, policy, {gang(std::vector<std::string>(8, "1g.5gb"), uid)}, {}, {0});
        EXPECT(more[0].verdict == Verdict::None);
        bool threw = false;
        try { r.PlaceGangs(list, policy, {gang({"1g.5gb"}, uid)}, {}, {1, 1}); }
        catch (const std::runtime_error&) { threw = true; }
        EXPECT(threw);
    }
    {   // with a locality per gang: a one-node gang of three 1g.5gb with minimum 2 on a node with two free slices
        InstasliceList list;
        list.Items.push_back(node("n0", {"GPU-0"}));
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_MIN_MEMBERS | ISL_FLAG_GANG_LOCALITY);
        r.Sync(list);
        const std::vector<GangOutcome> a = r.PlaceGangs(list, policy, {gang({"4g.20gb", "2g.10gb"}, uid)}, {ISL_GANG_ONE_NODE}, {0});
        EXPECT(a[0].verdict == Verdict::Placed && a[0].allocs.size() == 2);      // slices 0-3 and 4-5
        const std::vector<GangOutcome> b = r.PlaceGangs(list, policy, {gang({"1g.5gb", "1g.5gb", "1g.5gb"}, uid)}, {ISL_GANG_ONE_NODE}, {1});
        EXPECT(b[0].verdict == Verdict::Placed && b[0].allocs.size() == 1 && b[0].allocs[0].Start == 6);    // 1g.5gb starts at 0..6 only
    }
    bool refused = false;
    try { InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_MIN_MEMBERS | ISL_FLAG_ALL_NODES); }
    catch (const std::runtime_error&) { refused = true; }
    EXPECT(refused);
    printf("host mirror gang-min selftest: PASS\n");
    return 0;
}
