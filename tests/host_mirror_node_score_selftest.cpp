// Self-test of the C++ host mirror's InstasliceReconciler on a node-scoring engine (ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED): the
// first known-answer pair of tests/golden/kat_node_score.json on Instaslice objects, committed into the CRs.  Built and run by
// tests/test_gpu_node_score.py.
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "../instaslice_b200/host/instaslice_host.hpp"

using namespace instaslice;

#define EXPECT(cond)                                                             \
    do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); std::exit(1); } } while (0)

static std::vector<Mig> h100_80gb() {
    struct R { const char* n; int size; std::vector<int> starts; int gi; };
    const std::vector<R> rows = {{"1g.10gb", 1, {0, 1, 2, 3, 4, 5, 6}, 0}, {"1g.20gb", 2, {0, 2, 4, 6}, 9}, {"2g.20gb", 2, {0, 2, 4}, 1},
                                 {"3g.40gb", 4, {0, 4}, 2},                {"4g.40gb", 4, {0}, 3},           {"7g.80gb", 8, {0}, 4}};
    std::vector<Mig> out;
    for (const R& r : rows) {
        Mig m; m.Profile = r.n; m.Giprofileid = r.gi; m.CIProfileID = r.gi; m.CIEngProfileID = 0;
        for (int s : r.starts) m.Placements.push_back({r.size, s});
        out.push_back(m);
    }
    return out;
}

// node n0: one empty GPU; node n1: two GPUs with slices 0-3 allocated (occupancy 0x0F each)
static InstasliceList cluster() {
    InstasliceList list;
    Instaslice a; a.Name = "n0"; a.Spec.Migplacement = h100_80gb(); a.Spec.MigGPUUUID["GPU-0"] = "NVIDIA H100 80GB HBM3";
    Instaslice b; b.Name = "n1"; b.Spec.Migplacement = h100_80gb();
    for (const char* g : {"GPU-1", "GPU-2"}) {
        b.Spec.MigGPUUUID[g] = "NVIDIA H100 80GB HBM3";
        AllocationDetails d; d.PodUUID = std::string("old-") + g; d.GPUUUID = g; d.Start = 0; d.Size = 4; d.Allocationstatus = "created";
        b.Spec.Allocations[d.PodUUID] = d;
    }
    list.Items.push_back(a);
    list.Items.push_back(b);
    return list;
}

int main() {
    FirstFitPolicy packer;      // the allocation-policy hook packs AllocationDetails; the engine policy chooses the node
    {   // MostAllocated: n0 scores 100 x 1 / 8 = 12, n1 100 x 9 / 16 = 56
        InstasliceList list = cluster();
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 12, 1u << 12, ISL_POLICY_MOST_ALLOCATED);
        r.Sync(list);
        const std::vector<Outcome> out = r.PlacePending(list, packer, {PendingPod{Pod{"p0", "default", "p0"}, "1g.10gb"}});
        EXPECT(out.size() == 1 && out[0].verdict == Verdict::Placed);
        EXPECT(out[0].alloc.Nodename == "n1" && out[0].alloc.GPUUUID == "GPU-1" && out[0].alloc.Start == 4 && out[0].alloc.Size == 1);
        EXPECT(list.Items[1].Spec.Allocations.count("p0") == 1 && list.Items[0].Spec.Allocations.empty());
    }
    {   // LeastAllocated: n0 scores 100 x 7 / 8 = 87, n1 100 x 7 / 16 = 43
        InstasliceList list = cluster();
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 12, 1u << 12, ISL_POLICY_LEAST_ALLOCATED);
        r.Sync(list);
        const std::vector<Outcome> out = r.PlacePending(list, packer, {PendingPod{Pod{"p0", "default", "p0"}, "1g.10gb"}});
        EXPECT(out.size() == 1 && out[0].verdict == Verdict::Placed);
        EXPECT(out[0].alloc.Nodename == "n0" && out[0].alloc.GPUUUID == "GPU-0" && out[0].alloc.Start == 0 && out[0].alloc.Size == 1);
        EXPECT(list.Items[0].Spec.Allocations.count("p0") == 1);
    }
    printf("PASS\n");
    return 0;
}
