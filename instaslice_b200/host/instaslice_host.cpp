// instaslice_host.cpp — see instaslice_host.hpp.  Builds into instaslice_b200/libislhost.so (links libislplace.so).
#include "instaslice_host.hpp"

#include <algorithm>
#include <set>
#include <stdexcept>

namespace instaslice {

const char* const kErrNoGpu = "failed to find allocatable gpu";

static void check(int rc, isl_engine* h, const char* what) {
    if (rc != ISL_OK) throw std::runtime_error(std::string(what) + ": " + isl_strerror(rc) + (rc == ISL_ECUDA ? std::string(" ") + isl_last_cuda_error(h) : ""));
}

AllocationDetails FirstFitPolicy::SetAllocationDetails(const std::string& profileName, uint32_t newStart, uint32_t size, const std::string& podUUID,
                                                       const std::string& nodename, const std::string& processed, int gi, int ci, int cieng,
                                                       const std::string& ns, const std::string& podName, const std::string& gpuUuid) {
    AllocationDetails a;
    a.Profile = profileName; a.Start = newStart; a.Size = size; a.PodUUID = podUUID; a.Nodename = nodename; a.Allocationstatus = processed;
    a.Giprofileid = gi; a.CIProfileID = ci; a.CIEngProfileID = cieng; a.Namespace = ns; a.PodName = podName; a.GPUUUID = gpuUuid;
    return a;
}

InstasliceReconciler::InstasliceReconciler(uint32_t quirks, uint32_t max_gpus, uint32_t max_batch, uint32_t policy, uint32_t flags) {
    isl_config cfg{};
    cfg.abi_version = ISL_ABI_VERSION; cfg.policy = policy; cfg.quirks = quirks; cfg.device = -1;
    cfg.max_gpus = max_gpus; cfg.max_batch = max_batch; cfg.flags = flags;
    check(isl_create(&cfg, &h_), nullptr, "isl_create");
}
InstasliceReconciler::~InstasliceReconciler() { if (h_) isl_destroy(h_); }

uint8_t InstasliceReconciler::occupancyByte(const Instaslice& is, const std::string& gpuUUID) {
    uint32_t busy = 0;
    for (const auto& kv : is.Spec.Prepared) {                       // :312-320
        const PreparedDetails& p = kv.second;
        if (p.Parent == gpuUUID && p.PodUUID.empty()) {
            if (p.Start + p.Size > ISL_SLOTS) throw std::runtime_error("prepared span beyond slice 7 (reference panics, :316)");
            busy |= ((1u << p.Size) - 1u) << p.Start;
        }
    }
    for (const auto& kv : is.Spec.Allocations) {                    // :322-328, any status
        const AllocationDetails& a = kv.second;
        if (a.GPUUUID == gpuUUID) {
            if (a.Start + a.Size > ISL_SLOTS) throw std::runtime_error("allocation span beyond slice 7 (reference panics, :325)");
            busy |= ((1u << a.Size) - 1u) << a.Start;
        }
    }
    return (uint8_t)busy;
}

void InstasliceReconciler::extractGpuProfile(const Instaslice& is, const std::string& profileName, int* size, int* gi, int* ci, int* cieng) {
    *size = *gi = *ci = *cieng = 0;
    for (const Mig& m : is.Spec.Migplacement)                       // the LAST matching row wins, size of its first placement
        if (m.Profile == profileName && !m.Placements.empty()) { *size = m.Placements[0].Size; *gi = m.Giprofileid; *ci = m.CIProfileID; *cieng = m.CIEngProfileID; }
}

void InstasliceReconciler::Sync(const InstasliceList& list) {
    if (list.Items.empty()) throw std::runtime_error("no Instaslice objects");
    // every node publishes its own Migplacement (instaslice_daemonset.go:588-664): group identical tables, name index = first appearance
    auto same = [](const std::vector<Mig>& a, const std::vector<Mig>& b) {
        if (a.size() != b.size()) return false;
        for (size_t i = 0; i < a.size(); ++i) {
            if (a[i].Profile != b[i].Profile || a[i].Giprofileid != b[i].Giprofileid || a[i].Placements.size() != b[i].Placements.size()) return false;
            for (size_t k = 0; k < a[i].Placements.size(); ++k)
                if (a[i].Placements[k].Size != b[i].Placements[k].Size || a[i].Placements[k].Start != b[i].Placements[k].Start) return false;
        }
        return true;
    };
    std::vector<const std::vector<Mig>*> tables;
    nodeTable_.clear();
    profiles_.clear();
    for (const Instaslice& is : list.Items) {
        size_t t = 0;
        while (t < tables.size() && !same(*tables[t], is.Spec.Migplacement)) ++t;
        if (t == tables.size()) {
            if (tables.size() >= ISL_MAX_TABLES) throw std::runtime_error("more than 8 distinct per-node profile tables");
            tables.push_back(&is.Spec.Migplacement);
            for (const Mig& m : is.Spec.Migplacement) {
                if (m.Placements.empty()) throw std::runtime_error("profile " + m.Profile + " has no placements (reference panics, :334)");
                if (!profiles_.count(m.Profile)) { const uint8_t idx = (uint8_t)profiles_.size(); profiles_[m.Profile] = idx; }
            }
        }
        nodeTable_.push_back((uint8_t)t);
    }
    if (profiles_.size() > ISL_MAX_PROFILES) throw std::runtime_error("too many profile names");
    const size_t P = profiles_.size();
    std::vector<isl_profile> rows(tables.size() * P);          // rows[t * P + name]; n_starts == 0: no row of that name in table t
    for (size_t t = 0; t < tables.size(); ++t) {
        std::map<std::string, bool> seen;
        for (const Mig& m : *tables[t]) {                       // FIRST row with a name serves the start search (:332-340)
            if (seen[m.Profile]) continue;
            seen[m.Profile] = true;
            isl_profile r{};
            r.size = (uint8_t)m.Placements[0].Size;
            for (const Placement& p : m.Placements) {
                bool dup = false;
                for (uint32_t k = 0; k < r.n_starts; ++k) dup = dup || r.starts[k] == p.Start;
                if (!dup && r.n_starts < ISL_MAX_STARTS) r.starts[r.n_starts++] = (uint8_t)p.Start;
            }
            r.gi_profile_id = m.Giprofileid; r.ci_profile_id = m.CIProfileID; r.ci_eng_profile_id = m.CIEngProfileID;
            rows[t * P + profiles_[m.Profile]] = r;
        }
    }
    nTables_ = (uint32_t)tables.size();
    gpuUUID_.clear(); gpuNode_.clear(); gpuIndex_.clear(); nodeOff_.assign(1, 0); orphans_ = false;
    std::vector<uint8_t> occ;
    for (size_t n = 0; n < list.Items.size(); ++n) {
        const Instaslice& is = list.Items[n];
        for (const auto& kv : is.Spec.MigGPUUUID) {                 // std::map: ascending UUID = canonical order (SURVEY Q6)
            gpuIndex_[kv.first] = (uint32_t)gpuUUID_.size();
            gpuUUID_.push_back(kv.first); gpuNode_.push_back(n);
            occ.push_back(occupancyByte(is, kv.first));
        }
        nodeOff_.push_back((uint32_t)gpuUUID_.size());
        for (const auto& kv : is.Spec.Prepared)
            if (!kv.second.PodUUID.empty() && !is.Spec.Allocations.count(kv.second.PodUUID)) orphans_ = true;
    }
    if (gpuUUID_.empty()) throw std::runtime_error("no GPUs");
    check(isl_load_profile_tables(h_, nTables_, (uint32_t)P, rows.data()), h_, "isl_load_profile_tables");
    check(isl_load_inventory(h_, (uint32_t)list.Items.size(), nodeOff_.data(), occ.data()), h_, "isl_load_inventory");
    check(isl_set_node_tables(h_, (uint32_t)nodeTable_.size(), nodeTable_.data()), h_, "isl_set_node_tables");
}

void InstasliceReconciler::UpdateNode(const InstasliceList& list, size_t node) {
    if (node + 1 >= nodeOff_.size()) { Sync(list); return; }
    const Instaslice& is = list.Items[node];
    const uint32_t lo = nodeOff_[node], hi = nodeOff_[node + 1];
    if (is.Spec.MigGPUUUID.size() != hi - lo) { Sync(list); return; }
    std::vector<uint8_t> occ;
    uint32_t g = lo;
    for (const auto& kv : is.Spec.MigGPUUUID) {
        if (kv.first != gpuUUID_[g++]) { Sync(list); return; }
        occ.push_back(occupancyByte(is, kv.first));
    }
    check(isl_write_occupancy(h_, lo, (uint32_t)occ.size(), occ.data()), h_, "isl_write_occupancy");
    orphans_ = false;
    for (const Instaslice& it : list.Items)
        for (const auto& kv : it.Spec.Prepared)
            if (!kv.second.PodUUID.empty() && !it.Spec.Allocations.count(kv.second.PodUUID)) orphans_ = true;
}

uint32_t InstasliceReconciler::getStartIndexFromPreparedState(const Instaslice& is, const std::string& gpuUUID, const std::string& profileName) {
    auto it = profiles_.find(profileName);
    if (it == profiles_.end()) return ISL_START_NONE;
    const uint8_t occ = occupancyByte(is, gpuUUID);
    uint8_t start = ISL_START_NONE;
    uint32_t table = 0;                                         // the table of the node that owns the GPU
    auto gi = gpuIndex_.find(gpuUUID);
    if (gi != gpuIndex_.end()) table = nodeTable_[gpuNode_[gi->second]];
    check(isl_eval_starts(h_, it->second | (table << 8), 1, &occ, &start), h_, "isl_eval_starts");
    return start;
}

std::vector<isl_request> InstasliceReconciler::requests(const std::vector<std::string>& names) const {
    std::vector<isl_request> req(names.size());
    for (size_t i = 0; i < names.size(); ++i) {
        auto it = profiles_.find(names[i]);
        req[i] = isl_request{(uint32_t)i, it == profiles_.end() ? (uint8_t)ISL_PROFILE_UNKNOWN : it->second, (uint8_t)ISL_OP_ALLOC, 0, 0};
    }
    return req;
}

std::vector<isl_result> InstasliceReconciler::place(const std::vector<std::string>& names, uint32_t lo, uint32_t hi) {
    std::vector<isl_request> req = requests(names);
    std::vector<isl_result> res(names.size());
    // restriction, placement and restore under ONE engine lock: nothing leaks when the call throws, two callers cannot interleave
    check(isl_place_batch_range(h_, lo, hi, (uint32_t)req.size(), req.data(), res.data()), h_, "isl_place_batch_range");
    return res;
}

void InstasliceReconciler::releaseSpan(const isl_result& r) {
    isl_span s{r.gpu, r.start, r.size, 0};
    check(isl_free_batch(h_, 1, &s), h_, "isl_free_batch");
}

bool InstasliceReconciler::findDeviceForASlice(const InstasliceList& list, size_t node, const std::string& profileName, AllocationPolicy& policy,
                                               const Pod& pod, AllocationDetails* out, std::string* err) {
    const std::vector<isl_result> res = place({profileName}, nodeOff_[node], nodeOff_[node + 1]);
    if (res[0].status != ISL_ST_PLACED) { if (err) *err = kErrNoGpu; return false; }
    releaseSpan(res[0]);
    const Instaslice& is = list.Items[node];
    int size, gi, ci, cieng;
    extractGpuProfile(is, profileName, &size, &gi, &ci, &cieng);
    *out = policy.SetAllocationDetails(profileName, res[0].start, (uint32_t)size, pod.UID, is.Name, "creating", gi, ci, cieng, pod.Namespace, pod.Name,
                                       gpuUUID_[res[0].gpu]);
    return true;
}

AllocationDetails InstasliceReconciler::pack(const InstasliceList& list, AllocationPolicy& policy, const PendingPod& p, const isl_result& r) {
    const Instaslice& is = list.Items[gpuNode_[r.gpu]];
    int size, gi, ci, cieng;
    extractGpuProfile(is, p.ProfileName, &size, &gi, &ci, &cieng);
    return policy.SetAllocationDetails(p.ProfileName, r.start, (uint32_t)size, p.pod.UID, is.Name, "creating", gi, ci, cieng, p.pod.Namespace,
                                       p.pod.Name, gpuUUID_[r.gpu]);
}

bool InstasliceReconciler::vetoed(const InstasliceList& list, const isl_result& r, const AllocationDetails& a) const {
    for (const auto& kv : list.Items[gpuNode_[r.gpu]].Spec.Prepared) {     // :198-203 exact-match veto
        const PreparedDetails& item = kv.second;
        if (item.Parent == a.GPUUUID && item.Size == a.Size && item.Start == a.Start) return true;
    }
    return false;
}

Outcome InstasliceReconciler::commitOrVeto(InstasliceList& list, AllocationPolicy& policy, const PendingPod& p, const isl_result& r) {
    Outcome o;
    o.alloc = pack(list, policy, p, r);
    if (vetoed(list, r, o.alloc)) {
        releaseSpan(r);
        o.verdict = Verdict::Veto;
        return o;
    }
    list.Items[gpuNode_[r.gpu]].Spec.Allocations[p.pod.UID] = o.alloc;     // :215-219 (r.Update)
    o.verdict = Verdict::Placed;
    return o;
}

std::vector<GangOutcome> InstasliceReconciler::PlaceGangs(InstasliceList& list, AllocationPolicy& policy, const std::vector<std::vector<PendingPod>>& gangs) {
    return PlaceGangs(list, policy, gangs, {});
}

// `locality` empty: every ALLOC keeps start 0, which an engine without ISL_FLAG_GANG_LOCALITY ignores
std::vector<GangOutcome> InstasliceReconciler::PlaceGangs(InstasliceList& list, AllocationPolicy& policy, const std::vector<std::vector<PendingPod>>& gangs,
                                                          const std::vector<uint8_t>& locality) {
    return PlaceGangs(list, policy, gangs, locality, {});
}

// `minMembers` empty: every ALLOC keeps size 0, which an engine without ISL_FLAG_GANG_MIN_MEMBERS ignores
std::vector<GangOutcome> InstasliceReconciler::PlaceGangs(InstasliceList& list, AllocationPolicy& policy, const std::vector<std::vector<PendingPod>>& gangs,
                                                          const std::vector<uint8_t>& locality, const std::vector<uint8_t>& minMembers) {
    std::vector<GangOutcome> out(gangs.size());
    if (!locality.empty() && locality.size() != gangs.size()) throw std::runtime_error("one locality per gang");
    if (!minMembers.empty() && minMembers.size() != gangs.size()) throw std::runtime_error("one minimum per gang");
    if (gangs.empty()) return out;
    if (orphans_ && gangs.size() > 1) {         // the veto must see one gang at a time: a vetoed gang leaves no trace before the next
        auto one = [](const std::vector<uint8_t>& v, size_t g) { return v.empty() ? std::vector<uint8_t>{} : std::vector<uint8_t>{v[g]}; };
        for (size_t g = 0; g < gangs.size(); ++g) out[g] = PlaceGangs(list, policy, {gangs[g]}, one(locality, g), one(minMembers, g))[0];
        return out;
    }
    std::vector<std::string> names;
    std::vector<uint32_t> off{0};
    for (const auto& gang : gangs) {
        if (gang.empty()) throw std::runtime_error("empty gang");
        for (const PendingPod& p : gang) names.push_back(p.ProfileName);
        off.push_back((uint32_t)names.size());
    }
    std::vector<isl_request> req = requests(names);
    if (!locality.empty())
        for (size_t g = 0; g < gangs.size(); ++g)
            for (uint32_t i = off[g]; i < off[g + 1]; ++i) req[i].start = locality[g];
    if (!minMembers.empty())
        for (size_t g = 0; g < gangs.size(); ++g)
            for (uint32_t i = off[g]; i < off[g + 1]; ++i) req[i].size = minMembers[g];
    std::vector<isl_result> res(names.size());
    check(isl_place_gangs(h_, (uint32_t)gangs.size(), off.data(), req.data(), res.data()), h_, "isl_place_gangs");
    for (size_t g = 0; g < gangs.size(); ++g) {
        // the placed pods are a leading run: the whole gang, none, or an elastic gang's first pods
        uint32_t end = off[g];
        while (end < off[g + 1] && res[end].status == ISL_ST_PLACED) ++end;
        if (end == off[g]) continue;            // nothing of the gang was committed
        bool veto = false;
        GangOutcome& o = out[g];
        for (uint32_t i = off[g]; i < end; ++i) {
            o.allocs.push_back(pack(list, policy, gangs[g][i - off[g]], res[i]));
            veto = veto || vetoed(list, res[i], o.allocs.back());
        }
        if (veto) {                             // one member vetoed: every span of the gang is released again
            for (uint32_t i = off[g]; i < end; ++i) releaseSpan(res[i]);
            o.allocs.clear();
            o.verdict = Verdict::Veto;
            continue;
        }
        for (uint32_t i = off[g]; i < end; ++i) list.Items[gpuNode_[res[i].gpu]].Spec.Allocations[gangs[g][i - off[g]].pod.UID] = o.allocs[i - off[g]];
        o.verdict = Verdict::Placed;
    }
    return out;
}

// Dense ranks over the pending pods' values `own` and every value of podPriority, the victims in (GPU, start) order and their pod UIDs.
void InstasliceReconciler::preemptVictims(const InstasliceList& list, const std::vector<int32_t>& own,
                                          const std::map<std::string, int32_t>& podPriority, std::map<int32_t, uint8_t>& rank,
                                          std::vector<isl_victim>& victims, std::vector<std::string>& uids) const {
    std::set<int32_t> values(own.begin(), own.end());
    for (const auto& kv : podPriority) values.insert(kv.second);
    if (values.size() > 255) throw std::runtime_error("more than 255 distinct priority values");
    for (int32_t v : values) rank.emplace(v, (uint8_t)rank.size());
    auto span = [](uint32_t start, uint32_t size) { return ((1u << size) - 1u) << start; };
    for (uint32_t g = 0; g < gpuUUID_.size(); ++g) {            // victims in (GPU, start) order
        const InstasliceSpec& spec = list.Items[gpuNode_[g]].Spec;
        const std::string& uuid = gpuUUID_[g];
        std::vector<uint32_t> masks;                            // every entry that marks slices of this GPU busy (:306-328)
        for (const auto& kv : spec.Prepared)
            if (kv.second.Parent == uuid && kv.second.PodUUID.empty()) masks.push_back(span(kv.second.Start, kv.second.Size));
        std::vector<std::pair<uint32_t, std::string>> allocs;
        for (const auto& kv : spec.Allocations)
            if (kv.second.GPUUUID == uuid) { masks.push_back(span(kv.second.Start, kv.second.Size)); allocs.push_back({kv.second.Start, kv.first}); }
        std::sort(allocs.begin(), allocs.end());
        for (const auto& [start, uid] : allocs) {
            const AllocationDetails& a = spec.Allocations.at(uid);
            const auto pr = podPriority.find(uid);
            if (pr == podPriority.end() || a.Allocationstatus == "deleted") continue;
            const uint32_t m = span(a.Start, a.Size);
            int overlapping = 0;                                // itself once; anything more would keep its slices busy
            for (uint32_t x : masks) overlapping += (x & m) != 0;
            if (overlapping > 1) continue;
            victims.push_back({g, (uint8_t)a.Start, (uint8_t)a.Size, rank.at(pr->second), 0});
            uids.push_back(uid);
        }
    }
}

std::vector<PreemptOutcome> InstasliceReconciler::PreemptPending(const InstasliceList& list, const std::vector<PreemptPod>& pods,
                                                                 const std::map<std::string, int32_t>& podPriority) {
    std::vector<PreemptOutcome> out(pods.size());
    if (pods.empty()) return out;
    std::vector<int32_t> own;
    for (const PreemptPod& p : pods) own.push_back(p.Priority);
    std::map<int32_t, uint8_t> rank;
    std::vector<isl_victim> victims;
    std::vector<std::string> uids;
    preemptVictims(list, own, podPriority, rank, victims, uids);
    std::vector<std::string> names;
    std::vector<uint8_t> prio;
    for (const PreemptPod& p : pods) { names.push_back(p.ProfileName); prio.push_back(rank.at(p.Priority)); }
    const std::vector<isl_request> req = requests(names);
    std::vector<isl_result> res(pods.size());
    std::vector<uint32_t> evict(pods.size() * 8);
    check(isl_preempt(h_, (uint32_t)pods.size(), req.data(), prio.data(), (uint32_t)victims.size(), victims.data(), res.data(), evict.data()),
          h_, "isl_preempt");
    for (size_t i = 0; i < pods.size(); ++i) {
        if (res[i].status != ISL_ST_PLACED) continue;
        PreemptOutcome& o = out[i];
        o.Nodename = list.Items[gpuNode_[res[i].gpu]].Name;
        o.GPUUUID = gpuUUID_[res[i].gpu];
        o.Start = res[i].start; o.Size = res[i].size;
        for (size_t k = 0; k < 8; ++k) if (evict[i * 8 + k] != ISL_GPU_NONE) o.Victims.push_back(uids[evict[i * 8 + k]]);
        o.verdict = o.Victims.empty() ? PreemptVerdict::Fits : PreemptVerdict::Preempt;
    }
    return out;
}

std::vector<GangPreemptOutcome> InstasliceReconciler::PreemptPendingGangs(const InstasliceList& list,
                                                                          const std::vector<std::vector<PreemptPod>>& gangs,
                                                                          const std::map<std::string, int32_t>& podPriority,
                                                                          const std::vector<uint8_t>& locality) {
    std::vector<GangPreemptOutcome> out(gangs.size());
    if (!locality.empty() && locality.size() != gangs.size()) throw std::runtime_error("one locality per gang");
    std::vector<int32_t> own;
    std::vector<std::string> names;
    std::vector<uint32_t> gang_of;
    for (size_t k = 0; k < gangs.size(); ++k) {
        if (gangs[k].empty()) throw std::runtime_error("empty gang");
        for (const PreemptPod& p : gangs[k]) {
            if (p.Priority != gangs[k][0].Priority) throw std::runtime_error("the pods of one gang have different priorities");
            own.push_back(p.Priority); names.push_back(p.ProfileName); gang_of.push_back((uint32_t)k);
        }
    }
    if (names.empty()) return out;
    std::map<int32_t, uint8_t> rank;
    std::vector<isl_victim> victims;
    std::vector<std::string> uids;
    preemptVictims(list, own, podPriority, rank, victims, uids);
    std::vector<isl_request> req = requests(names);
    std::vector<uint8_t> prio;
    for (size_t i = 0; i < req.size(); ++i) {
        req[i].handle = gang_of[i];                                   // P1: a gang is a run of equal handles
        if (!locality.empty() && req[i].op == ISL_OP_ALLOC) req[i].start = locality[gang_of[i]];
        prio.push_back(rank.at(own[i]));
    }
    std::vector<isl_result> res(req.size());
    std::vector<uint32_t> evict(req.size() * 8);
    check(isl_preempt(h_, (uint32_t)req.size(), req.data(), prio.data(), (uint32_t)victims.size(), victims.data(), res.data(), evict.data()),
          h_, "isl_preempt");
    for (size_t i = 0, k = 0; k < gangs.size(); i += gangs[k].size(), ++k) {
        GangPreemptOutcome& o = out[k];
        bool all = true;
        for (size_t j = i; j < i + gangs[k].size(); ++j) all &= res[j].status == ISL_ST_PLACED;
        if (!all) continue;
        std::set<uint32_t> gone;
        for (size_t j = i; j < i + gangs[k].size(); ++j) {
            PreemptOutcome w;
            w.verdict = PreemptVerdict::Fits;
            w.Nodename = list.Items[gpuNode_[res[j].gpu]].Name;
            w.GPUUUID = gpuUUID_[res[j].gpu];
            w.Start = res[j].start; w.Size = res[j].size;
            o.pods.push_back(w);
            for (size_t x = 0; x < 8; ++x) if (evict[j * 8 + x] != ISL_GPU_NONE) gone.insert(evict[j * 8 + x]);
        }
        for (uint32_t v : gone) o.Victims.push_back(uids[v]);
        o.verdict = o.Victims.empty() ? PreemptVerdict::Fits : PreemptVerdict::Preempt;
    }
    return out;
}

std::vector<Outcome> InstasliceReconciler::PlacePending(InstasliceList& list, AllocationPolicy& policy, const std::vector<PendingPod>& pods) {
    std::vector<Outcome> out(pods.size());
    if (pods.empty()) return out;
    if (orphans_ && pods.size() > 1) {          // the veto must see one pod at a time, exactly like the reference
        for (size_t i = 0; i < pods.size(); ++i) out[i] = PlacePending(list, policy, {pods[i]})[0];
        return out;
    }
    std::vector<std::string> names;
    for (const PendingPod& p : pods) names.push_back(p.ProfileName);
    const std::vector<isl_result> res = place(names, 0, (uint32_t)gpuUUID_.size());
    for (size_t i = 0; i < pods.size(); ++i)
        if (res[i].status == ISL_ST_PLACED) out[i] = commitOrVeto(list, policy, pods[i], res[i]);
    return out;
}

bool InstasliceReconciler::Release(InstasliceList& list, const std::string& podUID) {
    for (size_t n = 0; n < list.Items.size(); ++n) {
        Instaslice& is = list.Items[n];
        auto it = is.Spec.Allocations.find(podUID);
        if (it == is.Spec.Allocations.end()) continue;
        is.Spec.Allocations.erase(it);
        // rebuild the node's bytes from the CR (OR over every remaining entry, :306-328) instead of clearing the span blindly:
        // slices another entry still covers stay busy, exactly what the reference's next rebuild would say
        UpdateNode(list, n);
        return true;
    }
    return false;
}

}  // namespace instaslice
