// Self-test of InstasliceReconciler::PlaceGangs (C++ host mirror) on node-scoring engines created with ISL_FLAG_GANG_NODE_SCORE, on a
// GPU: under MostAllocated a one-node gang joins the pod already running, under LeastAllocated it takes the empty node, distinct-node
// replicas spread, and the engine refuses the flag without a node-scoring policy and a locality flag under node scoring without the
// flag.  Built and run by tests/test_gpu_gang_score.py.
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
    for (uint32_t pol : {ISL_POLICY_MOST_ALLOCATED, ISL_POLICY_LEAST_ALLOCATED}) {
        // one call: a pod alone (a tie between two empty nodes goes to n0), then a job of two pods on one node, then two replicas on
        // distinct nodes through the per-gang locality
        InstasliceList list = cluster();
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 16, 1u << 16, pol, ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_LOCALITY);
        r.Sync(list);
        const std::vector<GangOutcome> out = r.PlaceGangs(list, policy, {gang({"1g.5gb"}, uid), gang({"1g.5gb", "1g.5gb"}, uid),
                                                                         gang({"2g.10gb", "2g.10gb"}, uid)},
                                                          {ISL_GANG_ANY_NODES, ISL_GANG_ONE_NODE, ISL_GANG_DISTINCT_NODES});
        EXPECT(out.size() == 3);
        for (const GangOutcome& o : out) EXPECT(o.verdict == Verdict::Placed);
        EXPECT(out[0].allocs[0].GPUUUID == "GPU-0" && out[0].allocs[0].Start == 0);
        if (pol == ISL_POLICY_MOST_ALLOCATED) {      // pack: the job joins the pod on n0
            EXPECT(out[1].allocs[0].GPUUUID == "GPU-0" && out[1].allocs[0].Start == 1);
            EXPECT(out[1].allocs[1].GPUUUID == "GPU-0" && out[1].allocs[1].Start == 2);
            // n0 is the fuller node (3 of 8 slices busy): the first replica goes there, at the first free 2g start; the second to n1
            EXPECT(out[2].allocs[0].GPUUUID == "GPU-0" && out[2].allocs[0].Start == 4);
            EXPECT(out[2].allocs[1].GPUUUID == "GPU-1" && out[2].allocs[1].Start == 0);
        } else {                                     // spread: the job takes the empty n1
            EXPECT(out[1].allocs[0].GPUUUID == "GPU-1" && out[1].allocs[0].Start == 0);
            EXPECT(out[1].allocs[1].GPUUUID == "GPU-1" && out[1].allocs[1].Start == 1);
            // n0 has 1 busy slice, n1 2: the first replica goes to n0, the second to n1
            EXPECT(out[2].allocs[0].GPUUUID == "GPU-0" && out[2].allocs[0].Start == 2);
            EXPECT(out[2].allocs[1].GPUUUID == "GPU-1" && out[2].allocs[1].Start == 2);
        }
        EXPECT(out[2].allocs[0].Nodename != out[2].allocs[1].Nodename);
        r.Sync(list);                                // the CR and the engine agree
    }
    EXPECT(refused(ISL_POLICY_FIRST_FIT, ISL_FLAG_GANG_NODE_SCORE));
    EXPECT(refused(ISL_POLICY_MOST_ALLOCATED, ISL_FLAG_GANG_ONE_NODE));
    EXPECT(refused(ISL_POLICY_LEAST_ALLOCATED, ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_FEW_NODES));
    EXPECT(!refused(ISL_POLICY_MOST_ALLOCATED, ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_ONE_NODE));
    printf("host mirror gang-score selftest: PASS\n");
    return 0;
}
