// instaslice_host.hpp — C++ host-side mirror of the reference's allocator interface over the C ABI.
//
// The reference controller is Go and no Go toolchain exists in this image, so the host side above
// include/islplace.h is written in C++ with the reference's names, argument meaning and error behaviour
// (internal/controller/instaslice_controller.go at b34e86d):
//   InstasliceReconciler::findDeviceForASlice            :240-262
//   InstasliceReconciler::getStartIndexFromPreparedState :303-384  (occupancy build :306-328 = occupancyByte)
//   InstasliceReconciler::extractGpuProfile              :283-300
//   AllocationPolicy / FirstFitPolicy / LeftToRightPolicy / RightToLeftPolicy  :48-56, :436-469
//   InstasliceReconciler::PlacePending                   node loop + Prepared veto of Reconcile :188-232, batched
//   InstasliceReconciler::PlaceGangs                     the same for all-or-nothing pod groups (extension: isl_place_gangs)
// Types follow api/v1alpha1/instaslice_types.go:23-72.  Nothing here decides a placement: every decision comes
// back from libislplace.so.  The Go twin of this file is integration/go/placement_engine.go.
#pragma once

#include <map>
#include <string>
#include <vector>

#include "../../include/islplace.h"

namespace instaslice {

struct Placement { int Size = 0; int Start = 0; };
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
    std::map<std::string, std::string> MigGPUUUID;
    std::map<std::string, AllocationDetails> Allocations;
    std::map<std::string, PreparedDetails> Prepared;
    std::vector<Mig> Migplacement;
};
struct Instaslice { std::string Name; InstasliceSpec Spec; };
struct InstasliceList { std::vector<Instaslice> Items; };
struct Pod { std::string UID, Namespace, Name; };

// :48-50 — the allocation-policy hook: packs, chooses nothing
struct AllocationPolicy {
    virtual ~AllocationPolicy() = default;
    virtual AllocationDetails SetAllocationDetails(const std::string& profileName, uint32_t newStart, uint32_t size, const std::string& podUUID,
                                                   const std::string& nodename, const std::string& processed, int discoveredGiprofile,
                                                   int Ciprofileid, int Ciengprofileid, const std::string& ns, const std::string& podName,
                                                   const std::string& gpuUuid) = 0;
};
struct FirstFitPolicy : AllocationPolicy {       // :436-453
    AllocationDetails SetAllocationDetails(const std::string&, uint32_t, uint32_t, const std::string&, const std::string&, const std::string&, int, int,
                                           int, const std::string&, const std::string&, const std::string&) override;
};
struct LeftToRightPolicy : AllocationPolicy {    // :456-461, a stub in the reference: empty AllocationDetails
    AllocationDetails SetAllocationDetails(const std::string&, uint32_t, uint32_t, const std::string&, const std::string&, const std::string&, int, int,
                                           int, const std::string&, const std::string&, const std::string&) override { return {}; }
};
struct RightToLeftPolicy : LeftToRightPolicy {}; // :464-469

enum class Verdict { Placed, None, Veto };       // allocation written / "failed to find allocatable gpu" everywhere / :198-203 requeue
struct PendingPod { Pod pod; std::string ProfileName; };
struct Outcome { Verdict verdict = Verdict::None; AllocationDetails alloc; };
// Priority preemption (extension: isl_preempt): a pending pod with the int32 value of its PriorityClass; the answer for it.
struct PreemptPod { Pod pod; std::string ProfileName; int32_t Priority = 0; };
enum class PreemptVerdict { Fits, Preempt, None };     // fits as things are / fits once Victims are gone / no GPU even with evictions
struct PreemptOutcome {
    PreemptVerdict verdict = PreemptVerdict::None;
    std::string Nodename, GPUUUID;                    // where the pod would go (Fits and Preempt)
    uint32_t Start = 0, Size = 0;
    std::vector<std::string> Victims;                 // pod UIDs to delete first (Preempt)
};
struct GangOutcome { Verdict verdict = Verdict::None; std::vector<AllocationDetails> allocs; };   // allocs: one per pod when Placed
// One gang of PreemptPendingGangs: where each pod would go (Fits and Preempt, one entry per pod; their Victims are empty) and the union of
// the pod UIDs to delete first (Preempt)
struct GangPreemptOutcome {
    PreemptVerdict verdict = PreemptVerdict::None;
    std::vector<PreemptOutcome> pods;
    std::vector<std::string> Victims;
};

extern const char* const kErrNoGpu;              // "failed to find allocatable gpu" (:261)

class InstasliceReconciler {
public:
    // policy: the engine's isl_config.policy, e.g. ISL_POLICY_MOST_ALLOCATED to pack MIG pods onto the fullest nodes or
    // ISL_POLICY_LEAST_ALLOCATED to spread them (include/islplace.h).  flags: isl_config.flags, e.g. ISL_FLAG_GANG_ONE_NODE so that
    // PlaceGangs puts every gang on one node, ISL_FLAG_GANG_DISTINCT_NODES so that it puts every member of a gang on a different node,
    // ISL_FLAG_GANG_FEW_NODES so that it puts a gang on one node when one takes it and on as few nodes as it greedily can otherwise, or
    // ISL_FLAG_GANG_LOCALITY so that PlaceGangs takes one of these localities per gang; ISL_FLAG_GANG_MIN_MEMBERS (alone or with one of
    // the four) so that PlaceGangs takes a minimum per gang; with a node-scoring policy, ISL_FLAG_GANG_NODE_SCORE (alone or with the
    // one-node, distinct-node or locality flag) so that PlaceGangs places gangs by the node score; with ISL_FLAG_GANG_LOCALITY,
    // ISL_FLAG_GANG_BALANCED so that a locality of ISL_GANG_BALANCED_NODES(maxSkew) spreads a gang over the nodes; with
    // ISL_FLAG_GANG_NODE_SCORE, ISL_FLAG_GANG_NODE_SCORE_ALL so that few-node, elastic and balanced gangs are node-scored as well
    explicit InstasliceReconciler(uint32_t quirks = ISL_QUIRKS_REF_EXACT, uint32_t max_gpus = 1u << 16, uint32_t max_batch = 1u << 16,
                                  uint32_t policy = ISL_POLICY_FIRST_FIT, uint32_t flags = 0);
    ~InstasliceReconciler();
    InstasliceReconciler(const InstasliceReconciler&) = delete;

    // Rebuild the flat inventory from the listed custom resources (the CR is the checkpoint).  Throws std::runtime_error
    // on what makes the reference panic (SURVEY Q7) and on engine errors.
    void Sync(const InstasliceList& list);
    // Incremental sync after ONE Instaslice object (list.Items[node]) changed: only that node's occupancy bytes are rewritten.
    // Falls back to Sync when the node's GPU set changed.
    void UpdateNode(const InstasliceList& list, size_t node);

    static uint8_t occupancyByte(const Instaslice& is, const std::string& gpuUUID);                        // :306-328
    uint32_t getStartIndexFromPreparedState(const Instaslice& is, const std::string& gpuUUID, const std::string& profileName);   // :303-384
    static void extractGpuProfile(const Instaslice& is, const std::string& profileName, int* size, int* gi, int* ci, int* cieng);  // :283-300
    // :240-262 — first GPU of ONE node; returns false and sets *err = kErrNoGpu when nothing fits.  Like the reference it
    // does not record the allocation (the tentative engine commit is released again).
    bool findDeviceForASlice(const InstasliceList& list, size_t node, const std::string& profileName, AllocationPolicy& policy, const Pod& pod,
                             AllocationDetails* out, std::string* err);
    // Reconcile's node loop for many gated pods in order, ONE engine call; allocations are written into `list`.
    std::vector<Outcome> PlacePending(InstasliceList& list, AllocationPolicy& policy, const std::vector<PendingPod>& pods);
    // All-or-nothing pod groups in order, ONE engine call (isl_place_gangs): a gang is Placed only when every pod of it got a slice, and
    // only then are its allocations written into `list`.  None: a pod found no GPU, nothing of the gang was committed.  Veto: the
    // Prepared exact-match check (:198-203) fired on a pod, every span of the gang was released again.  Empty gangs throw.
    std::vector<GangOutcome> PlaceGangs(InstasliceList& list, AllocationPolicy& policy, const std::vector<std::vector<PendingPod>>& gangs);
    // The same with one node locality per gang (ISL_GANG_ANY_NODES, _ONE_NODE, _FEW_NODES or _DISTINCT_NODES), for a reconciler created
    // with ISL_FLAG_GANG_LOCALITY, or ISL_GANG_BALANCED_NODES(maxSkew) under ISL_FLAG_GANG_BALANCED as well: one call places gangs of
    // every locality on one occupancy.  Throws unless there is one per gang.
    std::vector<GangOutcome> PlaceGangs(InstasliceList& list, AllocationPolicy& policy, const std::vector<std::vector<PendingPod>>& gangs,
                                        const std::vector<uint8_t>& locality);
    // The same with one minimum m (0..255) per gang as well (empty: none), for a reconciler created with ISL_FLAG_GANG_MIN_MEMBERS
    // (include/islplace.h M1-M7): a gang whose leading pods reach its minimum while a later pod finds no GPU is Placed with those pods
    // only, so its allocs are a shorter, leading part of the gang, and only they are written into `list`.  `locality` may be empty
    // on an engine without ISL_FLAG_GANG_LOCALITY.  Throws unless each non-empty list has one entry per gang.
    std::vector<GangOutcome> PlaceGangs(InstasliceList& list, AllocationPolicy& policy, const std::vector<std::vector<PendingPod>>& gangs,
                                        const std::vector<uint8_t>& locality, const std::vector<uint8_t>& minMembers);
    // Which lower-priority allocations each pending pod should evict, in order, ONE engine call (isl_preempt).  podPriority maps the UID
    // of each running pod to its PriorityClass value; values become dense ranks (more than 255 distinct values throw).  An allocation
    // may be evicted only when its pod's priority is known, its status is not "deleted" and no other entry that marks slices busy
    // overlaps it; every other busy slice is pinned.  Writes nothing into `list`: the caller deletes the Victims, and once their
    // allocations are gone a later PlacePending places the pod there.
    std::vector<PreemptOutcome> PreemptPending(const InstasliceList& list, const std::vector<PreemptPod>& pods,
                                               const std::map<std::string, int32_t>& podPriority);
    // The same for gangs that must all run or none, ONE engine call on an engine created with ISL_FLAG_GANG_PREEMPT (include/islplace.h
    // P1-P8): a gang gets victims for every pod or none.  The pods of one gang carry one priority (else it throws).  locality: empty, or
    // one ISL_GANG_* value per gang (0, 1 or 3) on an engine created with ISL_FLAG_GANG_LOCALITY as well.
    std::vector<GangPreemptOutcome> PreemptPendingGangs(const InstasliceList& list, const std::vector<std::vector<PreemptPod>>& gangs,
                                                        const std::map<std::string, int32_t>& podPriority,
                                                        const std::vector<uint8_t>& locality = {});
    // The daemonset removed Allocations[podUID] (instaslice_daemonset.go:261-263).
    bool Release(InstasliceList& list, const std::string& podUID);

private:
    isl_engine* h_ = nullptr;
    std::vector<std::string> gpuUUID_;
    std::vector<size_t> gpuNode_;
    std::vector<uint32_t> nodeOff_;
    std::vector<uint8_t> nodeTable_;      // per-node profile table (heterogeneous clusters)
    uint32_t nTables_ = 1;
    std::map<std::string, uint8_t> profiles_;
    std::map<std::string, uint32_t> gpuIndex_;
    bool orphans_ = false;
    void preemptVictims(const InstasliceList& list, const std::vector<int32_t>& own, const std::map<std::string, int32_t>& podPriority,
                        std::map<int32_t, uint8_t>& rank, std::vector<isl_victim>& victims, std::vector<std::string>& uids) const;
    std::vector<isl_request> requests(const std::vector<std::string>& names) const;
    std::vector<isl_result> place(const std::vector<std::string>& names, uint32_t lo, uint32_t hi);
    void releaseSpan(const isl_result& r);
    AllocationDetails pack(const InstasliceList& list, AllocationPolicy& policy, const PendingPod& p, const isl_result& r);
    bool vetoed(const InstasliceList& list, const isl_result& r, const AllocationDetails& a) const;
    Outcome commitOrVeto(InstasliceList& list, AllocationPolicy& policy, const PendingPod& p, const isl_result& r);
};

}  // namespace instaslice
