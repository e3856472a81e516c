// Self-test of InstasliceReconciler::PlaceGangs with balanced localities (C++ host mirror) on an engine created with
// ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_BALANCED, on a GPU: four replicas of one profile on two one-GPU nodes spread two and two at
// maxSkew 1, pack three and one at maxSkew 2, and go to the first GPU at maxSkew 4 (the gang's size), as any-node gangs do; a balanced
// byte on an engine without the flag is refused, and the engine refuses the flag without ISL_FLAG_GANG_LOCALITY.  Built and run by
// tests/test_gpu_gang_balance.py.
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

static std::vector<PendingPod> replicas(int n, int& uid) {
    std::vector<PendingPod> out;
    for (int i = 0; i < n; ++i) { out.push_back({Pod{"u" + std::to_string(uid), "default", "p" + std::to_string(uid)}, "1g.5gb"}); ++uid; }
    return out;
}

// the GPU of every allocation of one placed gang
static std::string gpus(const GangOutcome& o) {
    std::string s;
    for (const AllocationDetails& a : o.allocs) s += a.GPUUUID.back();
    return s;
}

int main() {
    FirstFitPolicy policy;
    int uid = 0;
    const uint32_t flags = ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_BALANCED;
    const char* want[] = {"0101", "0010", "0000"};          // maxSkew 1, 2 and 4: the header's worked example
    const uint8_t skews[] = {1, 2, 4};
    for (int k = 0; k < 3; ++k) {
        InstasliceList list;
        list.Items.push_back(node("n0", {"GPU-0"})); list.Items.push_back(node("n1", {"GPU-1"}));
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, flags);
        r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {replicas(4, uid)}, {(uint8_t)ISL_GANG_BALANCED_NODES(skews[k])});
        EXPECT(out.size() == 1 && out[0].verdict == Verdict::Placed && gpus(out[0]) == want[k]);
        EXPECT(list.Items[0].Spec.Allocations.size() + list.Items[1].Spec.Allocations.size() == 4);
        r.Sync(list);                                             // the CR and the engine agree
        // a distinct-node gang of three on two nodes has no room, and mixes with a balanced gang in one call
        const std::vector<GangOutcome> mixed = r.PlaceGangs(list, policy, {replicas(3, uid), replicas(2, uid)},
                                                            {ISL_GANG_DISTINCT_NODES, (uint8_t)ISL_GANG_BALANCED_NODES(1)});
        EXPECT(mixed[0].verdict == Verdict::None && mixed[1].verdict == Verdict::Placed && gpus(mixed[1]).size() == 2);
        EXPECT(gpus(mixed[1])[0] != gpus(mixed[1])[1]);
    }
    {   // without ISL_FLAG_GANG_BALANCED a byte above 3 is refused, and nothing is written
        InstasliceList list;
        list.Items.push_back(node("n0", {"GPU-0"})); list.Items.push_back(node("n1", {"GPU-1"}));
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_LOCALITY);
        r.Sync(list);
        bool threw = false;
        try { r.PlaceGangs(list, policy, {replicas(2, uid)}, {(uint8_t)ISL_GANG_BALANCED_NODES(1)}); }
        catch (const std::runtime_error&) { threw = true; }
        EXPECT(threw && list.Items[0].Spec.Allocations.empty() && list.Items[1].Spec.Allocations.empty());
    }
    bool refused = false;
    try { InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_BALANCED); }
    catch (const std::runtime_error&) { refused = true; }
    EXPECT(refused);
    printf("host mirror gang-balance selftest: PASS\n");
    return 0;
}
