// Self-test of the C++ host mirror's InstasliceReconciler with profile alternatives (ISL_FLAG_FIRST_AVAILABLE): the worked example of
// include/islplace.h (reference-exact quirks) on Instaslice objects, each pod's Fallbacks after its ProfileName, committed into the CRs
// under the chosen profile.  Built and run by tests/test_gpu_first_available.py.
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
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

static void allocate(Instaslice& is, const char* uid, const char* gpu, int start, int size) {
    AllocationDetails d; d.PodUUID = uid; d.GPUUUID = gpu; d.Start = start; d.Size = size; d.Allocationstatus = "created";
    is.Spec.Allocations[uid] = d;
}

// node n0: GPU-0 with slices 0-3 allocated (0x0F); node n1: GPU-1 with slices 0-5 allocated (0x3F)
static InstasliceList cluster() {
    InstasliceList list;
    Instaslice a; a.Name = "n0"; a.Spec.Migplacement = h100_80gb(); a.Spec.MigGPUUUID["GPU-0"] = "NVIDIA H100 80GB HBM3";
    allocate(a, "old-0", "GPU-0", 0, 4);
    Instaslice b; b.Name = "n1"; b.Spec.Migplacement = h100_80gb(); b.Spec.MigGPUUUID["GPU-1"] = "NVIDIA H100 80GB HBM3";
    allocate(b, "old-1", "GPU-1", 0, 4);
    allocate(b, "old-2", "GPU-1", 4, 2);
    list.Items.push_back(a);
    list.Items.push_back(b);
    return list;
}

static std::vector<PendingPod> pods() {
    return {PendingPod{Pod{"p0", "default", "p0"}, "3g.40gb", {"2g.20gb"}},
            PendingPod{Pod{"p1", "default", "p1"}, "3g.40gb", {"2g.20gb", "1g.10gb"}},
            PendingPod{Pod{"p2", "default", "p2"}, "2g.20gb", {"1g.10gb"}}};
}

int main() {
    FirstFitPolicy packer;
    {   // the worked example under reference-exact quirks: 2g.20gb at (0, 4), 1g.10gb at (0, 6), 1g.10gb at (1, 6)
        InstasliceList list = cluster();
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 12, 1u << 12, ISL_POLICY_FIRST_FIT, ISL_FLAG_FIRST_AVAILABLE);
        r.Sync(list);
        const std::vector<Outcome> out = r.PlacePending(list, packer, pods());
        EXPECT(out.size() == 3);
        for (const Outcome& o : out) EXPECT(o.verdict == Verdict::Placed);
        EXPECT(out[0].alloc.Profile == "2g.20gb" && out[0].alloc.GPUUUID == "GPU-0" && out[0].alloc.Start == 4 && out[0].alloc.Size == 2);
        EXPECT(out[0].alloc.Giprofileid == 1 && out[0].alloc.CIProfileID == 1);
        EXPECT(out[1].alloc.Profile == "1g.10gb" && out[1].alloc.GPUUUID == "GPU-0" && out[1].alloc.Start == 6 && out[1].alloc.Size == 1);
        EXPECT(out[1].alloc.Giprofileid == 0);
        EXPECT(out[2].alloc.Profile == "1g.10gb" && out[2].alloc.GPUUUID == "GPU-1" && out[2].alloc.Start == 6 && out[2].alloc.Size == 1);
        EXPECT(list.Items[0].Spec.Allocations.at("p0").Profile == "2g.20gb" && list.Items[1].Spec.Allocations.count("p2") == 1);
    }
    {   // an engine without the flag refuses fallbacks, and places pods without them as before
        InstasliceList list = cluster();
        InstasliceReconciler r(ISL_QUIRKS_REF_EXACT, 1u << 12, 1u << 12, ISL_POLICY_FIRST_FIT);
        r.Sync(list);
        bool thrown = false;
        try { r.PlacePending(list, packer, pods()); } catch (const std::invalid_argument&) { thrown = true; }
        EXPECT(thrown && list.Items[0].Spec.Allocations.size() == 1);
        const std::vector<Outcome> out = r.PlacePending(list, packer, {PendingPod{Pod{"p3", "default", "p3"}, "2g.20gb"}});
        EXPECT(out[0].verdict == Verdict::Placed && out[0].alloc.GPUUUID == "GPU-0" && out[0].alloc.Start == 4);
    }
    printf("PASS\n");
    return 0;
}
