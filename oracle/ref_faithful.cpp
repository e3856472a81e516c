// ref_faithful.cpp — structure-for-structure CPU restatement of the reference allocator.
//
// TEST INFRASTRUCTURE (see oracle.h).  PARITY UNPINNED by reference tests; pinned by
// SURVEY.md 8c known-answer vectors and by agreement with ref_fast.cpp / ref_py.py.
//
// Follows, in the reference tree (commit b34e86d):
//   internal/controller/instaslice_controller.go
//     :188-232  Reconcile's node loop and the Prepared exact-match veto
//     :240-262  findDeviceForASlice
//     :283-300  extractGpuProfile
//     :303-384  getStartIndexFromPreparedState
//     :436-453  FirstFitPolicy.SetAllocationDetails
//   api/v1alpha1/instaslice_types.go :23-72  (Mig, Placement, AllocationDetails, PreparedDetails, InstasliceSpec)
//
// The data structures are deliberately the reference's: string-keyed maps per node object,
// 36-character identifiers, occupancy rebuilt from Prepared + Allocations for every GPU of
// every node on every pod.  That cost profile IS the baseline being timed.
//
// Canonicalisation of the two non-deterministic iteration orders (SURVEY Q6): Go ranges over
// map[string]string MigGPUUUID in random order and over the informer cache's node list; here
// nodes are visited by index and GPUs by ascending UUID (std::map order); the generators name
// GPUs so that UUID order == canonical index order.

#include "oracle.h"

#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

namespace {

// ---- api/v1alpha1 types (instaslice_types.go:23-72) -------------------------------------
struct Placement { int Size; int Start; };
struct Mig {
    std::vector<Placement> Placements;
    std::string Profile;
    int Giprofileid = 0, CIProfileID = 0, CIEngProfileID = 0;
};
struct AllocationDetails {
    std::string Profile;
    uint32_t Start = 0, Size = 0;
    std::string PodUUID, GPUUUID, Nodename, Allocationstatus;
    int Giprofileid = 0, CIProfileID = 0, CIEngProfileID = 0;
    std::string Namespace, PodName;
};
struct PreparedDetails {
    std::string Profile;
    uint32_t Start = 0, Size = 0;
    std::string Parent, PodUUID;
    uint32_t Giinfoid = 0, Ciinfoid = 0;
};
struct InstasliceSpec {
    std::map<std::string, std::string> MigGPUUUID;            // uuid -> model name
    std::map<std::string, AllocationDetails> Allocations;     // podUID -> allocation
    std::map<std::string, PreparedDetails> Prepared;          // MIG uuid -> realised slice
    std::vector<Mig> Migplacement;
};
struct Instaslice { std::string Name; InstasliceSpec Spec; };
struct Pod { std::string UID, Namespace, Name; };

// ---- the "allocation-policy hook" (:48-50, :436-453): packs, chooses nothing --------------
struct AllocationPolicy {
    virtual ~AllocationPolicy() {}
    virtual AllocationDetails SetAllocationDetails(const std::string& profileName, uint32_t newStart, uint32_t size,
                                                   const std::string& podUUID, const std::string& nodename,
                                                   const std::string& processed, int gi, int ci, int cieng,
                                                   const std::string& ns, const std::string& podName,
                                                   const std::string& gpuUuid) = 0;
};
struct FirstFitPolicy : AllocationPolicy {
    AllocationDetails SetAllocationDetails(const std::string& profileName, uint32_t newStart, uint32_t size,
                                           const std::string& podUUID, const std::string& nodename,
                                           const std::string& processed, int gi, int ci, int cieng,
                                           const std::string& ns, const std::string& podName,
                                           const std::string& gpuUuid) override {
        AllocationDetails a;
        a.Profile = profileName; a.Start = newStart; a.Size = size; a.PodUUID = podUUID;
        a.Nodename = nodename; a.Allocationstatus = processed; a.Giprofileid = gi;
        a.CIProfileID = ci; a.CIEngProfileID = cieng; a.Namespace = ns; a.PodName = podName;
        a.GPUUUID = gpuUuid;
        return a;
    }
};

constexpr uint32_t kNotValidIndex = 9;   // :248, :343

// getStartIndexFromPreparedState (:303-384).  `quirks` selects the reference's exact bounds
// behaviour (REF_EXACT) or the repaired one (FIXED); the structure of the scan is unchanged.
uint32_t getStartIndexFromPreparedState(const Instaslice& is, const std::string& gpuUUID,
                                        const std::string& profileName, uint32_t quirks) {
    uint32_t busy[ISL_SLOTS];
    for (uint32_t i = 0; i < ISL_SLOTS; ++i) busy[i] = 0;                       // :306-310
    for (const auto& kv : is.Spec.Prepared) {                                   // :312-320
        const PreparedDetails& item = kv.second;
        if (item.Parent == gpuUUID && item.PodUUID.empty())
            for (uint32_t i = 0; i < item.Size; ++i) busy[item.Start + i] = 1;
    }
    for (const auto& kv : is.Spec.Allocations) {                                // :322-328 (any status)
        const AllocationDetails& item = kv.second;
        if (item.GPUUUID == gpuUUID)
            for (uint32_t i = 0; i < item.Size; ++i) busy[item.Start + i] = 1;
    }
    int needed = 0;
    std::vector<int> starts;                                                    // :330-340 (fresh slice per call)
    for (const Mig& m : is.Spec.Migplacement) {
        if (m.Profile == profileName) {
            needed = m.Placements[0].Size;
            for (const Placement& p : m.Placements) starts.push_back(p.Start);
            break;
        }
    }
    const bool strict = quirks & ISL_QUIRK_STRICT_BOUND;
    const bool pow2   = quirks & ISL_QUIRK_POW2_ONLY;
    uint32_t newStart = kNotValidIndex;                                         // :343
    for (int v : starts) {                                                      // :344-381
        if (busy[v] != 0) continue;
        if (needed == 1) { newStart = (uint32_t)v; break; }
        const bool handled = pow2 ? (needed == 2 || needed == 4 || needed == 8) : (needed >= 2 && needed <= 8);
        if (!handled) continue;                                                 // Q2: e.g. size 3 never places
        const bool inside = strict ? (v + needed < (int)ISL_SLOTS) : (v + needed <= (int)ISL_SLOTS);
        if (!inside) continue;                                                  // Q1
        bool all_free = true;
        for (int i = 0; i < needed; ++i) all_free = all_free && busy[v + i] == 0;
        if (!all_free) continue;
        newStart = (uint32_t)v;
        if (needed == 8 && strict) continue;  // :368-378 has no break; unreachable anyway under Q1
        break;
    }
    return newStart;
}

// extractGpuProfile (:283-300): the LAST matching Migplacement row wins, first placement's size.
void extractGpuProfile(const Instaslice& is, const std::string& profileName, int* size, int* gi, int* ci, int* cieng) {
    *size = *gi = *ci = *cieng = 0;
    for (const Mig& m : is.Spec.Migplacement) {
        if (m.Profile != profileName) continue;
        if (!m.Placements.empty()) {
            *size = m.Placements[0].Size; *gi = m.Giprofileid; *ci = m.CIProfileID; *cieng = m.CIEngProfileID;
        }
    }
}

// findDeviceForASlice (:240-262)
bool findDeviceForASlice(Instaslice& is, const std::string& profileName, AllocationPolicy& policy,
                         const Pod& pod, uint32_t quirks, AllocationDetails* out) {
    for (const auto& kv : is.Spec.MigGPUUUID) {                                 // :242 (canonical: ascending UUID)
        const std::string& gpuuuid = kv.first;
        uint32_t newStart = getStartIndexFromPreparedState(is, gpuuuid, profileName, quirks);
        if (newStart == kNotValidIndex) continue;                               // :248-252
        int size, gi, ci, cieng;
        extractGpuProfile(is, profileName, &size, &gi, &ci, &cieng);            // :253
        *out = policy.SetAllocationDetails(profileName, newStart, (uint32_t)size, pod.UID, is.Name, "creating",
                                           gi, ci, cieng, pod.Namespace, pod.Name, gpuuuid);   // :254-256
        return true;
    }
    return false;                                                               // :261 "failed to find allocatable gpu"
}

std::string fmt(const char* f, unsigned long long v) { char b[64]; snprintf(b, sizeof b, f, v); return b; }

}  // namespace

struct orc_faithful {
    std::vector<Instaslice> items;              // InstasliceList.Items in canonical node order
    std::vector<uint32_t> node_off;
    std::vector<std::string> profile_names;     // row index -> name used in the CRD rows
    std::vector<std::string> gpu_uuid;          // canonical index -> UUID
    std::vector<uint32_t> gpu_node;
    uint32_t quirks = ISL_QUIRKS_REF_EXACT;
    uint64_t next_pod = 0;                      // pod ids for ALLOC requests: pod-<n>
    uint64_t next_mig = 0;
    // (gpu,start,size) -> podUID of the Allocations entry, so a FREE request can name a span
    std::map<uint64_t, std::string> span_owner;
    std::map<uint64_t, std::string> span_prepared;
    FirstFitPolicy policy;
    static uint64_t span_key(uint32_t gpu, uint32_t start, uint32_t size) { return ((uint64_t)gpu << 8) | (start << 4) | (size & 15); }
};

extern "C" {

orc_faithful* orc_f_new_tables(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows_all,
                               const uint8_t* node_table, uint32_t quirks);
orc_faithful* orc_f_new(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_profiles, const isl_profile* rows, uint32_t quirks) {
    return orc_f_new_tables(n_nodes, node_off, 1, n_profiles, rows, nullptr, quirks);
}
// Every node publishes its OWN Migplacement (instaslice_daemonset.go:588-664): node n gets the rows of table node_table[n].
orc_faithful* orc_f_new_tables(uint32_t n_nodes, const uint32_t* node_off, uint32_t n_tables, uint32_t n_profiles, const isl_profile* rows_all,
                               const uint8_t* node_table, uint32_t quirks) {
    (void)n_tables;
    orc_faithful* h = new orc_faithful;
    h->quirks = quirks;
    h->node_off.assign(node_off, node_off + n_nodes + 1);
    const uint32_t G = node_off[n_nodes];
    h->gpu_uuid.resize(G); h->gpu_node.resize(G);
    for (uint32_t p = 0; p < n_profiles; ++p) h->profile_names.push_back(fmt("%llug.row", p));
    h->items.resize(n_nodes);
    for (uint32_t n = 0; n < n_nodes; ++n) {
        Instaslice& is = h->items[n];
        is.Name = fmt("node-%08llu", n);
        for (uint32_t g = node_off[n]; g < node_off[n + 1]; ++g) {
            // 40-char UUID like NVML's "GPU-xxxxxxxx-xxxx-xxxx-xxxx-xxxxxxxxxxxx"; ordered by canonical index
            h->gpu_uuid[g] = fmt("GPU-00000000-0000-0000-0000-%012llu", g);
            h->gpu_node[g] = n;
            is.Spec.MigGPUUUID[h->gpu_uuid[g]] = "NVIDIA A100-SXM4-40GB";
        }
        const isl_profile* rows = rows_all + (size_t)(node_table ? node_table[n] : 0) * n_profiles;
        for (uint32_t p = 0; p < n_profiles; ++p) {                 // one Mig row per profile (daemonset :642-658)
            if (rows[p].n_starts == 0) continue;                    // Placements[0] on an empty list panics (:334, Q7): never emitted
            Mig m; m.Profile = h->profile_names[p];
            m.Giprofileid = rows[p].gi_profile_id; m.CIProfileID = rows[p].ci_profile_id; m.CIEngProfileID = rows[p].ci_eng_profile_id;
            for (uint32_t s = 0; s < rows[p].n_starts; ++s) m.Placements.push_back({(int)rows[p].size, (int)rows[p].starts[s]});
            is.Spec.Migplacement.push_back(m);
        }
    }
    return h;
}
void orc_f_delete(orc_faithful* h) { delete h; }

int orc_f_add_prepared(orc_faithful* h, uint32_t gpu, uint32_t start, uint32_t size, int64_t pod_id) {
    if (gpu >= h->gpu_uuid.size() || size == 0 || start + size > ISL_SLOTS) return ISL_EINVAL;   // the reference would panic (Q7)
    PreparedDetails p; p.Start = start; p.Size = size; p.Parent = h->gpu_uuid[gpu];
    if (pod_id >= 0) p.PodUUID = fmt("pod-%032llu", (unsigned long long)pod_id);
    std::string key = fmt("MIG-00000000-0000-0000-0000-%012llu", h->next_mig++);
    h->items[h->gpu_node[gpu]].Spec.Prepared[key] = p;
    if (pod_id < 0) h->span_prepared[orc_faithful::span_key(gpu, start, size)] = key;
    return ISL_OK;
}
int orc_f_add_allocation(orc_faithful* h, uint32_t gpu, uint32_t start, uint32_t size, uint64_t pod_id) {
    if (gpu >= h->gpu_uuid.size() || size == 0 || start + size > ISL_SLOTS) return ISL_EINVAL;
    AllocationDetails a; a.Start = start; a.Size = size; a.GPUUUID = h->gpu_uuid[gpu];
    a.PodUUID = fmt("pod-%032llu", (unsigned long long)pod_id); a.Allocationstatus = "created";
    a.Nodename = h->items[h->gpu_node[gpu]].Name; a.Namespace = "default"; a.PodName = a.PodUUID;
    h->items[h->gpu_node[gpu]].Spec.Allocations[a.PodUUID] = a;
    h->span_owner[orc_faithful::span_key(gpu, start, size)] = a.PodUUID;
    if (pod_id >= h->next_pod) h->next_pod = pod_id + 1;
    return ISL_OK;
}

int orc_f_place(orc_faithful* h, uint32_t n, const isl_request* in, isl_result* out, int all_nodes) {
    const uint32_t G = (uint32_t)h->gpu_uuid.size();
    // canonical batch: FREEs first (an Allocations entry deleted by the daemonset, instaslice_daemonset.go:261-263)
    for (uint32_t i = 0; i < n; ++i) {
        if (in[i].op == ISL_OP_ALLOC) continue;
        if (in[i].op != ISL_OP_FREE) { out[i] = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NOOP}; continue; }   // NOOP and any unknown op
        const uint32_t g = in[i].handle, st = in[i].start, sz = in[i].size;
        if (g >= G || sz == 0 || st + sz > ISL_SLOTS) { out[i] = {g, (uint8_t)st, (uint8_t)sz, (uint16_t)ISL_ST_BAD_SPAN}; continue; }
        const uint64_t key = orc_faithful::span_key(g, st, sz);
        auto it = h->span_owner.find(key);
        if (it != h->span_owner.end()) {
            h->items[h->gpu_node[g]].Spec.Allocations.erase(it->second);
            h->span_owner.erase(it);
        } else {
            auto ip = h->span_prepared.find(key);
            if (ip != h->span_prepared.end()) { h->items[h->gpu_node[g]].Spec.Prepared.erase(ip->second); h->span_prepared.erase(ip); }
        }
        out[i] = {g, (uint8_t)st, (uint8_t)sz, (uint16_t)ISL_ST_FREED};
    }
    // then one Reconcile per pending pod, in order (:188-232)
    for (uint32_t i = 0; i < n; ++i) {
        if (in[i].op != ISL_OP_ALLOC) continue;
        isl_result r = {ISL_GPU_NONE, (uint8_t)ISL_START_NONE, 0, (uint16_t)ISL_ST_NO_CAPACITY};
        Pod pod; pod.UID = fmt("pod-%032llu", (unsigned long long)h->next_pod++); pod.Namespace = "default"; pod.Name = pod.UID;
        std::string profileName;
        if (in[i].profile < h->profile_names.size()) profileName = h->profile_names[in[i].profile];
        else { profileName = "unknown"; r.status = ISL_ST_BAD_PROFILE; }
        bool podHasNodeAllocation = false, veto = false;
        for (size_t nidx = 0; nidx < h->items.size() && !veto; ++nidx) {          // :190
            Instaslice& is = h->items[nidx];
            AllocationDetails a;
            if (!findDeviceForASlice(is, profileName, h->policy, pod, h->quirks, &a)) continue;   // :192-196
            for (const auto& kv : is.Spec.Prepared) {                           // :198-203 exact-match veto
                const PreparedDetails& item = kv.second;
                if (item.Parent == a.GPUUUID && item.Size == a.Size && item.Start == a.Start) { veto = true; break; }
            }
            if (veto) break;
            is.Spec.Allocations[pod.UID] = a;                                   // :218-219 (r.Update)
            // canonical GPU index back from the UUID (last 12 digits)
            uint32_t gidx = (uint32_t)strtoull(a.GPUUUID.c_str() + a.GPUUUID.size() - 12, nullptr, 10);
            h->span_owner[orc_faithful::span_key(gidx, a.Start, a.Size)] = pod.UID;
            if (!podHasNodeAllocation) r = {gidx, (uint8_t)a.Start, (uint8_t)a.Size, (uint16_t)ISL_ST_PLACED};
            podHasNodeAllocation = true;
            if (!all_nodes) break;      // canonical semantics: first node wins.  The reference has no break (Q5).
        }
        if (veto && !podHasNodeAllocation) r.status = ORC_ST_VETO_REQUEUE;
        if (!podHasNodeAllocation && in[i].profile < h->profile_names.size()) {
            // report the size the profile row would have used, like the engine does
            int size = 0, gi, ci, cieng;
            for (const Instaslice& is : h->items) { extractGpuProfile(is, profileName, &size, &gi, &ci, &cieng); if (size) break; }
            r.size = (uint8_t)size;
        }
        out[i] = r;
    }
    return ISL_OK;
}

// same shape as isl_place_batch / orc_fast_place (bench.py's C5 replay harness takes one placer signature)
int orc_f_place_batch(orc_faithful* h, uint32_t n, const isl_request* in, isl_result* out) { return orc_f_place(h, n, in, out, 0); }

void orc_f_occupancy(orc_faithful* h, uint8_t* out) {
    for (size_t g = 0; g < h->gpu_uuid.size(); ++g) {
        const Instaslice& is = h->items[h->gpu_node[g]];
        uint8_t b = 0;
        for (const auto& kv : is.Spec.Prepared)
            if (kv.second.Parent == h->gpu_uuid[g] && kv.second.PodUUID.empty())
                for (uint32_t i = 0; i < kv.second.Size; ++i) b |= (uint8_t)(1u << (kv.second.Start + i));
        for (const auto& kv : is.Spec.Allocations)
            if (kv.second.GPUUUID == h->gpu_uuid[g])
                for (uint32_t i = 0; i < kv.second.Size; ++i) b |= (uint8_t)(1u << (kv.second.Start + i));
        out[g] = b;
    }
}
uint64_t orc_f_num_allocations(orc_faithful* h) {
    uint64_t n = 0; for (auto& is : h->items) n += is.Spec.Allocations.size(); return n;
}

}  // extern "C"
