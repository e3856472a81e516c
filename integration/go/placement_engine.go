// placement_engine.go — the cgo shim a maintainer adds to internal/controller/ of project-codeflare/instaslice
// (commit b34e86d) to route the allocator through libislplace.so.  SOURCE ONLY: there is no Go toolchain in the
// build image of this repository, so this file has never been compiled here; it is written against
// include/islplace.h and mirrors instaslice_b200/controller.py, which IS exercised by the GPU tests.
//
// What stays exactly as it is: Reconcile's pod state machine, the CRD types, the daemonset, and the
// AllocationPolicy hook (policy.SetAllocationDetails still packs the AllocationDetails).  What changes:
// the body of findDeviceForASlice / getStartIndexFromPreparedState (instaslice_controller.go:240-262,
// 303-384) becomes one isl_place_batch call.
package controller

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -lislplace -lcudart
#include <stdlib.h>
#include "islplace.h"
*/
import "C"

import (
	"fmt"
	"reflect"
	"sort"
	"unsafe"

	inferencev1alpha1 "codeflare.dev/instaslice/api/v1alpha1"
	v1 "k8s.io/api/core/v1"
)

// PlacementEngine mirrors the listed Instaslice objects into the device-resident inventory.
type PlacementEngine struct {
	h        *C.isl_engine
	gpuUUID  []string          // canonical GPU index -> UUID
	gpuNode  []int             // canonical GPU index -> index into the Instaslice list
	profiles map[string]uint8  // profile name -> row index (FIRST Migplacement row with that name, :332-340)
	orphans  bool              // a realised slice outlived its allocation: the :198-203 veto can fire
	nodeOff  []C.uint32_t      // node index -> first canonical GPU index
	nodeMig  [][]inferencev1alpha1.Mig // the Migplacement each node had at the last Sync (UpdateNode compares)
}

// hasOrphans: a Prepared entry that names a pod whose Allocations entry is gone — the only state in which the exact-match
// veto (:198-203) can fire.  Recomputed by Sync AND by every UpdateNode.
func hasOrphans(list *inferencev1alpha1.InstasliceList) bool {
	for n := range list.Items {
		is := &list.Items[n]
		for _, p := range is.Spec.Prepared {
			if _, live := is.Spec.Allocations[p.PodUUID]; p.PodUUID != "" && !live {
				return true
			}
		}
	}
	return false
}

// Engine policies (isl_config.policy): which GPU, or which node, a pod goes to.  The AllocationPolicy hook still packs the answer.
const (
	PolicyFirstFit       = uint32(C.ISL_POLICY_FIRST_FIT)
	PolicyBestFit        = uint32(C.ISL_POLICY_BEST_FIT)
	PolicyRightToLeft    = uint32(C.ISL_POLICY_RIGHT_TO_LEFT)
	PolicyMinFrag        = uint32(C.ISL_POLICY_MIN_FRAG)
	PolicyMostAllocated  = uint32(C.ISL_POLICY_MOST_ALLOCATED)  // NodeResourcesFit MostAllocated: pack onto the fullest nodes
	PolicyLeastAllocated = uint32(C.ISL_POLICY_LEAST_ALLOCATED) // NodeResourcesFit LeastAllocated: spread over the emptiest nodes
)

// Engine flags (isl_config.flags) a controller may want.
const (
	FlagGangOneNode = uint32(C.ISL_FLAG_GANG_ONE_NODE) // PlaceGangs puts every gang on one node, the first in scan order that takes it
	// PlaceGangs puts every member of a gang on a different node, member by member (greedy: list the larger pods first), so that
	// one node failing does not take down every replica.  Not with FlagGangOneNode.
	FlagGangDistinctNodes = uint32(C.ISL_FLAG_GANG_DISTINCT_NODES)
	// PlaceGangs puts a gang on one node when one takes it whole, else on as few nodes as it greedily can: each round the node that
	// places the most of the remaining pods takes them.  Not with FlagGangOneNode or FlagGangDistinctNodes.
	FlagGangFewNodes = uint32(C.ISL_FLAG_GANG_FEW_NODES)
	// PlaceGangsWithLocality takes one of the Gang* localities per gang, so one call places every kind of gang on one occupancy.
	// Not with the three flags above.
	FlagGangLocality = uint32(C.ISL_FLAG_GANG_LOCALITY)
	// PlaceGangsElastic takes a minimum per gang: a gang whose leading pods reach it while a later pod finds no GPU is placed with
	// those pods only.  Alone or with one of the four flags above.
	FlagGangMinMembers = uint32(C.ISL_FLAG_GANG_MIN_MEMBERS)
	// PreemptPendingGangs picks the victims of whole gangs, or none for a gang that still cannot run.  Alone or with FlagGangOneNode,
	// FlagGangDistinctNodes or FlagGangLocality; not with FlagGangFewNodes or FlagGangMinMembers.
	FlagGangPreempt = uint32(C.ISL_FLAG_GANG_PREEMPT)
	// On a PolicyMostAllocated or PolicyLeastAllocated engine, PlaceGangs places gangs by the node score: alone (any node) or with
	// FlagGangOneNode, FlagGangDistinctNodes or FlagGangLocality (no few-node locality); not with FlagGangFewNodes or FlagGangMinMembers
	// unless FlagGangNodeScoreAll is set as well.
	FlagGangNodeScore = uint32(C.ISL_FLAG_GANG_NODE_SCORE)
	// With FlagGangLocality: a locality of GangBalancedNodes(maxSkew) spreads a gang's pods over the nodes within that maxSkew
	// (topologySpreadConstraints on kubernetes.io/hostname).  Under node scoring only with FlagGangNodeScoreAll.
	FlagGangBalanced = uint32(C.ISL_FLAG_GANG_BALANCED)
	// With FlagGangNodeScore: few-node gangs (FlagGangFewNodes or GangFewNodes), elastic gangs (FlagGangMinMembers) and balanced
	// gangs (FlagGangBalanced) are placed by the node score too, so a packing or spreading cluster needs no second engine for them.
	FlagGangNodeScoreAll = uint32(C.ISL_FLAG_GANG_NODE_SCORE_ALL)
)

// StGangTrimmed is the record status of a pod its elastic gang was placed without (isl_result.status, FlagGangMinMembers).
const StGangTrimmed = uint16(C.ISL_ST_GANG_TRIMMED)

// Node locality of one gang for PlaceGangsWithLocality (an engine created with FlagGangLocality).
const (
	GangAnyNodes      = uint8(C.ISL_GANG_ANY_NODES)      // pods anywhere, as on an engine without a gang flag
	GangOneNode       = uint8(C.ISL_GANG_ONE_NODE)       // every pod on one node (Kueue's required hostname topology)
	GangFewNodes      = uint8(C.ISL_GANG_FEW_NODES)      // one node when one has room, else as few as it greedily can (preferred)
	GangDistinctNodes = uint8(C.ISL_GANG_DISTINCT_NODES) // every pod on a different node
)

// GangBalancedNodes is the locality of a gang whose pods spread over the nodes within maxSkew (1..252) of each other, on an engine
// created with FlagGangLocality | FlagGangBalanced; ok is false outside 1..252.
func GangBalancedNodes(maxSkew int) (locality uint8, ok bool) {
	if maxSkew < 1 || maxSkew > 252 {
		return 0, false
	}
	return uint8(3 + maxSkew), true
}

func NewPlacementEngine(maxGPUs, maxBatch uint32) (*PlacementEngine, error) {
	return NewPlacementEngineWithPolicy(maxGPUs, maxBatch, PolicyFirstFit)
}

// NewPlacementEngineWithPolicy creates the engine with one of the Policy* values, e.g. PolicyMostAllocated so that the cluster
// autoscaler can drain the nodes MIG pods leave empty, or PolicyLeastAllocated to spread inference replicas.
func NewPlacementEngineWithPolicy(maxGPUs, maxBatch, policy uint32) (*PlacementEngine, error) {
	return NewPlacementEngineWithFlags(maxGPUs, maxBatch, policy, 0)
}

// NewPlacementEngineWithFlags also sets Flag* values, e.g. FlagGangOneNode so that the pods of a gang share a node (host shared memory
// instead of the network), FlagGangDistinctNodes so that the replicas of a deployment land on different nodes, or FlagGangFewNodes so
// that a gang shares a node when one has room and still runs on a few nodes when none has.  isl_create refuses each of the three flags
// with PolicyMostAllocated or PolicyLeastAllocated, and any two of them together.
func NewPlacementEngineWithFlags(maxGPUs, maxBatch, policy, flags uint32) (*PlacementEngine, error) {
	cfg := C.isl_config{abi_version: C.ISL_ABI_VERSION, policy: C.uint32_t(policy), quirks: C.ISL_QUIRKS_REF_EXACT,
		device: -1, max_gpus: C.uint32_t(maxGPUs), max_batch: C.uint32_t(maxBatch), flags: C.uint32_t(flags)}
	var h *C.isl_engine
	if rc := C.isl_create(&cfg, &h); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_create: %s", C.GoString(C.isl_strerror(rc)))
	}
	return &PlacementEngine{h: h}, nil
}

func (e *PlacementEngine) Close() { C.isl_destroy(e.h) }

// occupancyByte is instaslice_controller.go:306-328: dangling Prepared entries and every Allocations entry
// (any status) mark their slices.
func occupancyByte(is *inferencev1alpha1.Instaslice, gpuUUID string) (uint8, error) {
	var busy uint8
	for _, item := range is.Spec.Prepared {
		if item.Parent == gpuUUID && item.PodUUID == "" {
			if item.Start+item.Size > 8 {
				return 0, fmt.Errorf("prepared span beyond slice 7")
			}
			busy |= uint8(((1 << item.Size) - 1) << item.Start)
		}
	}
	for _, item := range is.Spec.Allocations {
		if item.GPUUUID == gpuUUID {
			if item.Start+item.Size > 8 {
				return 0, fmt.Errorf("allocation span beyond slice 7")
			}
			busy |= uint8(((1 << item.Size) - 1) << item.Start)
		}
	}
	return busy, nil
}

// Sync rebuilds the flat inventory from the custom resources (the CR is the checkpoint).  Canonical order:
// nodes in list order, GPUs by ascending UUID inside a node (the reference's orders are random, :85, :242).
func (e *PlacementEngine) Sync(list *inferencev1alpha1.InstasliceList) error {
	if len(list.Items) == 0 {
		return fmt.Errorf("no Instaslice objects")
	}
	// every node publishes its OWN Migplacement (instaslice_daemonset.go:588-664): group identical tables (<= 8), profile NAME
	// index = order of first appearance; rows[t*P + name] with n_starts == 0 when table t has no row of that name
	type tableT = []inferencev1alpha1.Mig
	tables := []tableT{}
	nodeTable := make([]C.uint8_t, len(list.Items))
	e.profiles = map[string]uint8{}
	for n := range list.Items {
		mig := list.Items[n].Spec.Migplacement
		t := 0
		for ; t < len(tables); t++ {
			if reflect.DeepEqual(tables[t], tableT(mig)) {
				break
			}
		}
		if t == len(tables) {
			if len(tables) >= int(C.ISL_MAX_TABLES) {
				return fmt.Errorf("more than %d distinct per-node profile tables", int(C.ISL_MAX_TABLES))
			}
			tables = append(tables, mig)
			for _, m := range mig {
				if len(m.Placements) == 0 {
					return fmt.Errorf("profile %s has no placements", m.Profile) // the reference panics at :334
				}
				if _, ok := e.profiles[m.Profile]; !ok {
					e.profiles[m.Profile] = uint8(len(e.profiles))
				}
			}
		}
		nodeTable[n] = C.uint8_t(t)
	}
	P := len(e.profiles)
	if P == 0 {
		return fmt.Errorf("no node publishes a Migplacement row") // nothing could ever be placed; &rows[0] below would panic
	}
	rows := make([]C.isl_profile, len(tables)*P)
	for t, mig := range tables {
		seenName := map[string]bool{}
		for _, m := range mig {
			if seenName[m.Profile] { // the start search uses the FIRST row with a name (:332-340)
				continue
			}
			seenName[m.Profile] = true
			r := &rows[t*P+int(e.profiles[m.Profile])]
			r.size = C.uint8_t(m.Placements[0].Size)
			seen := map[int]bool{}
			for _, p := range m.Placements {
				if !seen[p.Start] {
					seen[p.Start] = true
					r.starts[r.n_starts] = C.uint8_t(p.Start)
					r.n_starts++
				}
			}
			r.gi_profile_id, r.ci_profile_id, r.ci_eng_profile_id = C.int32_t(m.Giprofileid), C.int32_t(m.CIProfileID), C.int32_t(m.CIEngProfileID)
		}
	}
	nodeOff := []C.uint32_t{0}
	occ := []C.uint8_t{}
	e.gpuUUID, e.gpuNode, e.nodeMig = nil, nil, nil
	e.orphans = hasOrphans(list)
	for n := range list.Items {
		e.nodeMig = append(e.nodeMig, list.Items[n].Spec.Migplacement)
		is := &list.Items[n]
		uuids := make([]string, 0, len(is.Spec.MigGPUUUID))
		for u := range is.Spec.MigGPUUUID {
			uuids = append(uuids, u)
		}
		sort.Strings(uuids)
		for _, u := range uuids {
			b, err := occupancyByte(is, u)
			if err != nil {
				return err
			}
			occ = append(occ, C.uint8_t(b))
			e.gpuUUID = append(e.gpuUUID, u)
			e.gpuNode = append(e.gpuNode, n)
		}
		nodeOff = append(nodeOff, C.uint32_t(len(e.gpuUUID)))
	}
	if len(occ) == 0 {
		return fmt.Errorf("no GPU in any Instaslice object")
	}
	if rc := C.isl_load_profile_tables(e.h, C.uint32_t(len(tables)), C.uint32_t(P), &rows[0]); rc != C.ISL_OK {
		return fmt.Errorf("isl_load_profile_tables: %s", C.GoString(C.isl_strerror(rc)))
	}
	if rc := C.isl_load_inventory(e.h, C.uint32_t(len(list.Items)), &nodeOff[0], &occ[0]); rc != C.ISL_OK {
		return fmt.Errorf("isl_load_inventory: %s", C.GoString(C.isl_strerror(rc)))
	}
	if rc := C.isl_set_node_tables(e.h, C.uint32_t(len(list.Items)), &nodeTable[0]); rc != C.ISL_OK {
		return fmt.Errorf("isl_set_node_tables: %s", C.GoString(C.isl_strerror(rc)))
	}
	e.nodeOff = nodeOff
	return nil
}

// UpdateNode is the incremental sync after ONE Instaslice object changed (an Allocations / Prepared entry appeared or was
// deleted): only that node's occupancy bytes are rewritten (isl_write_occupancy) instead of re-listing the cluster (:85).
func (e *PlacementEngine) UpdateNode(list *inferencev1alpha1.InstasliceList, n int) error {
	if n >= len(e.nodeMig) || n+1 >= len(e.nodeOff) {
		return e.Sync(list) // a node appeared
	}
	is := &list.Items[n]
	lo, hi := int(e.nodeOff[n]), int(e.nodeOff[n+1])
	if len(is.Spec.MigGPUUUID) != hi-lo || hi == lo || !reflect.DeepEqual(e.nodeMig[n], is.Spec.Migplacement) {
		return e.Sync(list) // GPU set or profile table of the node changed
	}
	occ := make([]C.uint8_t, 0, hi-lo)
	for g := lo; g < hi; g++ {
		if _, ok := is.Spec.MigGPUUUID[e.gpuUUID[g]]; !ok {
			return e.Sync(list)
		}
		b, err := occupancyByte(is, e.gpuUUID[g])
		if err != nil {
			return err
		}
		occ = append(occ, C.uint8_t(b))
	}
	if rc := C.isl_write_occupancy(e.h, C.uint32_t(lo), C.uint32_t(len(occ)), &occ[0]); rc != C.ISL_OK {
		return fmt.Errorf("isl_write_occupancy: %s", C.GoString(C.isl_strerror(rc)))
	}
	e.orphans = hasOrphans(list)
	return nil
}

// PendingPod is one gated pod that has no allocation yet (Reconcile :148-187 already ran for it).
type PendingPod struct {
	Pod         *v1.Pod
	ProfileName string // r.extractProfileName(limits), :154
}

const errNoGpu = "failed to find allocatable gpu" // :261

// FindDeviceForASlice is the literal replacement of the call at instaslice_controller.go:192
//   allocDetails, err := r.findDeviceForASlice(&instaslice, profileName, policy, pod)
// for the node list.Items[n]: the first GPU of THAT node with a legal start (:240-262), packed by the unchanged policy hook.
// isl_place_batch_range restricts, places and restores under one engine lock.  Like the reference it does not record the
// allocation (:257 is commented out there): the tentative commit is rolled back by rebuilding the node's bytes from the CR.
func (r *InstasliceReconciler) FindDeviceForASlice(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, n int, profileName string,
	policy AllocationPolicy, pod *v1.Pod) (*inferencev1alpha1.AllocationDetails, error) {
	row, ok := e.profiles[profileName]
	if !ok {
		return nil, fmt.Errorf(errNoGpu)
	}
	req := (*C.isl_request)(C.malloc(C.sizeof_isl_request))
	res := (*C.isl_result)(C.malloc(C.sizeof_isl_result))
	if req == nil || res == nil {
		C.free(unsafe.Pointer(req))
		C.free(unsafe.Pointer(res))
		return nil, fmt.Errorf("out of memory")
	}
	defer C.free(unsafe.Pointer(req))
	defer C.free(unsafe.Pointer(res))
	*req = C.isl_request{handle: 0, profile: C.uint8_t(row), op: C.ISL_OP_ALLOC}
	if rc := C.isl_place_batch_range(e.h, e.nodeOff[n], e.nodeOff[n+1], 1, req, res); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_place_batch_range: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(e.h)))
	}
	if res.status != C.ISL_ST_PLACED {
		return nil, fmt.Errorf(errNoGpu)
	}
	is := &list.Items[n]
	size, gi, ci, cieng := r.extractGpuProfile(is, profileName)
	a := policy.SetAllocationDetails(profileName, uint32(res.start), uint32(size), string(pod.UID), is.Name, "creating",
		gi, ci, cieng, pod.Namespace, pod.Name, e.gpuUUID[int(res.gpu)])
	if err := e.UpdateNode(list, n); err != nil {
		return nil, err
	}
	return a, nil
}

// commitOrVeto packs one PLACED result with the unchanged policy hook and applies the exact-match Prepared veto (:198-203).
// A vetoed placement is rolled back by rebuilding the node's occupancy bytes from the CR (an OR over all entries, like
// :306-328 — never a blind clear: an overlapping span must not be freed early).  Used by PlacePending AND PlaceBacklog.
func (r *InstasliceReconciler) commitOrVeto(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	p PendingPod, res C.isl_result) (*inferencev1alpha1.AllocationDetails, error) {
	gpu := int(res.gpu)
	n := e.gpuNode[gpu]
	is := &list.Items[n]
	size, gi, ci, cieng := r.extractGpuProfile(is, p.ProfileName) // :283-300, unchanged
	a := policy.SetAllocationDetails(p.ProfileName, uint32(res.start), uint32(size), string(p.Pod.UID), is.Name, "creating",
		gi, ci, cieng, p.Pod.Namespace, p.Pod.Name, e.gpuUUID[gpu]) // :254-256, unchanged
	for _, item := range is.Spec.Prepared { // :198-203
		if item.Parent == a.GPUUUID && item.Size == a.Size && item.Start == a.Start {
			return nil, e.UpdateNode(list, n) // undo the tentative commit; the caller requeues after 1 s
		}
	}
	return a, nil
}

func (e *PlacementEngine) fillRequests(req []C.isl_request, pods []PendingPod, base int) {
	for i, p := range pods {
		row, ok := e.profiles[p.ProfileName]
		if !ok {
			row = C.ISL_PROFILE_UNKNOWN
		}
		req[base+i] = C.isl_request{handle: C.uint32_t(base + i), profile: C.uint8_t(row), op: C.ISL_OP_ALLOC}
	}
}

// PlacePending resolves the pods in order with ONE engine call and packs the answers with the unchanged policy
// hook.  result[i] == nil means "failed to find allocatable gpu" on every node (:261, :229-232: requeue) or a veto.
func (r *InstasliceReconciler) PlacePending(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	pods []PendingPod) ([]*inferencev1alpha1.AllocationDetails, error) {
	n := len(pods)
	out := make([]*inferencev1alpha1.AllocationDetails, n)
	if n == 0 {
		return out, nil
	}
	if e.orphans && n > 1 { // the exact-match veto (:198-203) must see one pod at a time
		for i := range pods {
			one, err := r.PlacePending(e, list, policy, pods[i:i+1])
			if err != nil {
				return nil, err
			}
			out[i] = one[0]
		}
		return out, nil
	}
	// C-allocated request/result arrays: no Go pointer is retained by the engine after the call returns
	reqP, resP := C.malloc(C.size_t(n)*C.sizeof_isl_request), C.malloc(C.size_t(n)*C.sizeof_isl_result)
	if reqP == nil || resP == nil {
		C.free(reqP)
		C.free(resP)
		return nil, fmt.Errorf("out of memory")
	}
	defer C.free(reqP)
	defer C.free(resP)
	req := (*[1 << 28]C.isl_request)(reqP)[:n:n]
	res := (*[1 << 28]C.isl_result)(resP)[:n:n]
	e.fillRequests(req, pods, 0)
	if rc := C.isl_place_batch(e.h, C.uint32_t(n), &req[0], &res[0]); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_place_batch: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(e.h)))
	}
	for i, p := range pods {
		if res[i].status != C.ISL_ST_PLACED {
			continue
		}
		a, err := r.commitOrVeto(e, list, policy, p, res[i])
		if err != nil {
			return nil, err
		}
		out[i] = a
	}
	return out, nil
}

// PlaceGangs resolves all-or-nothing pod groups (the replicas of one deployment, the workers of one job) in order with ONE
// engine call (isl_place_gangs).  result[g] holds one AllocationDetails per pod of gang g, or is nil when the gang was not placed:
// a pod found no GPU (nothing of the gang was committed; requeue), or the Prepared exact-match veto (:198-203) fired on a pod, in
// which case every node the gang touched is rebuilt from the CR, which holds none of its allocations.  As in PlacePending the
// caller writes the returned allocations (r.Update).  Empty gangs are an error.
func (r *InstasliceReconciler) PlaceGangs(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	gangs [][]PendingPod) ([][]*inferencev1alpha1.AllocationDetails, error) {
	return r.PlaceGangsWithLocality(e, list, policy, gangs, nil)
}

// PlaceGangsWithLocality is PlaceGangs with one Gang* locality per gang (nil: none), for an engine created with FlagGangLocality:
// a training job on one node, replicas on distinct nodes, a job on few nodes and free pods in one call.
func (r *InstasliceReconciler) PlaceGangsWithLocality(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	gangs [][]PendingPod, locality []uint8) ([][]*inferencev1alpha1.AllocationDetails, error) {
	return r.PlaceGangsElastic(e, list, policy, gangs, locality, nil)
}

// PlaceGangsElastic is PlaceGangsWithLocality with one minimum m (0..255) per gang as well (nil: none), for an engine created with
// FlagGangMinMembers (a PodGroup's minMember, Volcano's minAvailable, Kueue's PodSet minCount).  locality may be nil on an engine
// without FlagGangLocality.  A gang whose leading pods reach its minimum while a later pod finds no GPU gets the allocations of those
// pods only, a shorter slice than the gang; list the pods the job needs first, since the placed pods are always a leading run.
func (r *InstasliceReconciler) PlaceGangsElastic(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	gangs [][]PendingPod, locality []uint8, minMembers []uint8) ([][]*inferencev1alpha1.AllocationDetails, error) {
	out := make([][]*inferencev1alpha1.AllocationDetails, len(gangs))
	if locality != nil && len(locality) != len(gangs) {
		return nil, fmt.Errorf("one locality per gang")
	}
	if minMembers != nil && len(minMembers) != len(gangs) {
		return nil, fmt.Errorf("one minimum per gang")
	}
	if len(gangs) == 0 {
		return out, nil
	}
	n := 0
	for _, g := range gangs {
		if len(g) == 0 {
			return nil, fmt.Errorf("empty gang")
		}
		n += len(g)
	}
	if e.orphans && len(gangs) > 1 { // the exact-match veto (:198-203) must see one gang at a time
		for g := range gangs {
			var loc, mins []uint8
			if locality != nil {
				loc = locality[g : g+1]
			}
			if minMembers != nil {
				mins = minMembers[g : g+1]
			}
			one, err := r.PlaceGangsElastic(e, list, policy, gangs[g:g+1], loc, mins)
			if err != nil {
				return nil, err
			}
			out[g] = one[0]
		}
		return out, nil
	}
	reqP, resP := C.malloc(C.size_t(n)*C.sizeof_isl_request), C.malloc(C.size_t(n)*C.sizeof_isl_result)
	offP := C.malloc(C.size_t(len(gangs)+1) * 4)
	if reqP == nil || resP == nil || offP == nil {
		C.free(reqP)
		C.free(resP)
		C.free(offP)
		return nil, fmt.Errorf("out of memory")
	}
	defer C.free(reqP)
	defer C.free(resP)
	defer C.free(offP)
	req := (*[1 << 28]C.isl_request)(reqP)[:n:n]
	res := (*[1 << 28]C.isl_result)(resP)[:n:n]
	off := (*[1 << 28]C.uint32_t)(offP)[: len(gangs)+1 : len(gangs)+1]
	off[0] = 0
	for g, pods := range gangs {
		e.fillRequests(req, pods, int(off[g]))
		off[g+1] = off[g] + C.uint32_t(len(pods))
		if locality != nil {
			for i := off[g]; i < off[g+1]; i++ {
				req[i].start = C.uint8_t(locality[g])
			}
		}
		if minMembers != nil {
			for i := off[g]; i < off[g+1]; i++ {
				req[i].size = C.uint8_t(minMembers[g])
			}
		}
	}
	if rc := C.isl_place_gangs(e.h, C.uint32_t(len(gangs)), &off[0], &req[0], &res[0]); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_place_gangs: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(e.h)))
	}
	for g, pods := range gangs {
		gres := res[off[g]:off[g+1]]
		placed := 0 // a leading run: the whole gang, none, or an elastic gang's first pods
		for placed < len(gres) && gres[placed].status == C.ISL_ST_PLACED {
			placed++
		}
		if placed == 0 {
			continue
		}
		pods, gres = pods[:placed], gres[:placed]
		allocs := make([]*inferencev1alpha1.AllocationDetails, len(pods))
		vetoed := false
		for i, p := range pods {
			a, err := r.commitOrVeto(e, list, policy, p, gres[i])
			if err != nil {
				return nil, err
			}
			vetoed = vetoed || a == nil
			allocs[i] = a
		}
		if vetoed { // the whole gang goes: rebuild every node it touched
			for i := range gres {
				if err := e.UpdateNode(list, e.gpuNode[int(gres[i].gpu)]); err != nil {
					return nil, err
				}
			}
			continue
		}
		out[g] = allocs
	}
	return out, nil
}

// Release: the daemonset removed Allocations[podUID] from list.Items[n] (instaslice_daemonset.go:261-263).  The node's occupancy
// bytes are REBUILT from the CR (OR over every remaining Prepared / Allocations entry, :306-328) rather than cleared blindly: if
// another entry still covers part of the span, those slices stay busy — exactly what the reference's next rebuild would say.
func (e *PlacementEngine) Release(list *inferencev1alpha1.InstasliceList, n int) error {
	return e.UpdateNode(list, n)
}

// hostArrays returns mapped pinned request / result arrays from the engine's own allocator (isl_host_alloc) or, when that
// fails, plain C.malloc'ed ones (pageable works for isl_place_stream, without the copy / delivery overlap).
func hostArrays(total int) (req []C.isl_request, res []C.isl_result, pinned bool, free func(), err error) {
	reqP, resP := C.isl_host_alloc(C.size_t(total)*C.sizeof_isl_request), C.isl_host_alloc(C.size_t(total)*C.sizeof_isl_result)
	pinned = reqP != nil && resP != nil
	if pinned {
		free = func() { C.isl_host_free(reqP); C.isl_host_free(resP) }
	} else {
		C.isl_host_free(reqP)
		C.isl_host_free(resP)
		reqP, resP = C.malloc(C.size_t(total)*C.sizeof_isl_request), C.malloc(C.size_t(total)*C.sizeof_isl_result)
		if reqP == nil || resP == nil {
			C.free(reqP)
			C.free(resP)
			return nil, nil, false, nil, fmt.Errorf("out of memory")
		}
		free = func() { C.free(reqP); C.free(resP) }
	}
	return (*[1 << 28]C.isl_request)(reqP)[:total:total], (*[1 << 28]C.isl_result)(resP)[:total:total], pinned, free, nil
}

// PlaceBacklog resolves several ordered batches (e.g. per-namespace queues drained in turn) with ONE isl_place_stream
// call: identical answers to PlacePending batch after batch, pipelined on the device.  With pinned arrays the engine copies
// batch b while it already places batch b-1 and writes finished chunks straight into `res`.
func (r *InstasliceReconciler) PlaceBacklog(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	batches [][]PendingPod) ([][]*inferencev1alpha1.AllocationDetails, error) {
	total := 0
	sizes := make([]C.uint32_t, len(batches))
	for b, pods := range batches {
		sizes[b] = C.uint32_t(len(pods))
		total += len(pods)
	}
	out := make([][]*inferencev1alpha1.AllocationDetails, len(batches))
	if total == 0 || e.orphans { // the exact-match veto (:198-203) needs one pod at a time: fall back to PlacePending
		for b, pods := range batches {
			one, err := r.PlacePending(e, list, policy, pods)
			if err != nil {
				return nil, err
			}
			out[b] = one
		}
		return out, nil
	}
	req, res, _, free, err := hostArrays(total)
	if err != nil {
		return nil, err
	}
	defer free()
	i := 0
	for _, pods := range batches {
		e.fillRequests(req, pods, i)
		i += len(pods)
	}
	if rc := C.isl_place_stream(e.h, C.uint32_t(len(batches)), &sizes[0], &req[0], &res[0]); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_place_stream: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(e.h)))
	}
	i = 0
	for b, pods := range batches {
		out[b] = make([]*inferencev1alpha1.AllocationDetails, len(pods))
		for k, p := range pods {
			if res[i].status == C.ISL_ST_PLACED { // same packing and the same :198-203 check as PlacePending
				a, err := r.commitOrVeto(e, list, policy, p, res[i])
				if err != nil {
					return nil, err
				}
				out[b][k] = a
			}
			i++
		}
	}
	return out, nil
}

// BacklogStream is the causal feed: batches are handed over WHILE earlier ones are still being placed, and the results of a
// batch can be read as soon as Wait(ticket) returns — the reconciler composes the next batch (e.g. re-queues pods whose
// allocation a deleted pod just released) from results it has already seen.  One persistent device kernel serves the whole
// stream (isl_stream_open / _submit / _wait / _close); results equal PlacePending batch after batch.
type BacklogStream struct {
	e    *PlacementEngine
	pods [][]PendingPod
	res  [][]C.isl_result
	free []func()
}

// inFlight: how many batches this caller keeps in flight (it Waits for batch b - inFlight before it Submits batch b).  1..3 tells the
// engine to resolve every batch by speculative rounds (all inventory stages at once, DESIGN.md 4.5) instead of pipelining different
// batches over the stages; 0 = no promise (deep backlogs).
func (e *PlacementEngine) OpenBacklogStream(maxBatches int, inFlight int) (*BacklogStream, error) {
	if e.orphans {
		return nil, fmt.Errorf("realised slices without allocation present: resolve pods one by one (PlacePending)")
	}
	if rc := C.isl_set_causal_window(e.h, C.uint32_t(inFlight)); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_set_causal_window: %s", C.GoString(C.isl_strerror(rc)))
	}
	if rc := C.isl_stream_open(e.h, C.uint32_t(maxBatches)); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_stream_open: %s", C.GoString(C.isl_strerror(rc)))
	}
	return &BacklogStream{e: e}, nil
}

// Submit enqueues one batch and returns its ticket at once.
func (s *BacklogStream) Submit(pods []PendingPod) (int, error) {
	req, res, pinned, free, err := hostArrays(len(pods))
	if err != nil {
		return -1, err
	}
	if !pinned { // the running kernel writes the results: they must live in mapped pinned memory
		free()
		return -1, fmt.Errorf("isl_host_alloc failed")
	}
	s.e.fillRequests(req, pods, 0)
	var ticket C.uint32_t
	if rc := C.isl_stream_submit(s.e.h, C.uint32_t(len(pods)), &req[0], &res[0], &ticket); rc != C.ISL_OK {
		free()
		return -1, fmt.Errorf("isl_stream_submit: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(s.e.h)))
	}
	s.pods, s.res, s.free = append(s.pods, pods), append(s.res, res), append(s.free, free)
	return int(ticket), nil
}

// Wait blocks until the batch's results are in host memory and packs them exactly like PlacePending.
func (s *BacklogStream) Wait(r *InstasliceReconciler, list *inferencev1alpha1.InstasliceList, policy AllocationPolicy,
	ticket int) ([]*inferencev1alpha1.AllocationDetails, error) {
	if rc := C.isl_stream_wait(s.e.h, C.uint32_t(ticket)); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_stream_wait: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(s.e.h)))
	}
	out := make([]*inferencev1alpha1.AllocationDetails, len(s.pods[ticket]))
	for k, p := range s.pods[ticket] {
		if s.res[ticket][k].status != C.ISL_ST_PLACED {
			continue
		}
		// the veto cannot fire here (no orphans at open; a veto rollback would need the engine, which the stream owns): pack only
		gpu := int(s.res[ticket][k].gpu)
		is := &list.Items[s.e.gpuNode[gpu]]
		size, gi, ci, cieng := r.extractGpuProfile(is, p.ProfileName)
		out[k] = policy.SetAllocationDetails(p.ProfileName, uint32(s.res[ticket][k].start), uint32(size), string(p.Pod.UID), is.Name, "creating",
			gi, ci, cieng, p.Pod.Namespace, p.Pod.Name, s.e.gpuUUID[gpu])
	}
	return out, nil
}

func (s *BacklogStream) Close() error {
	rc := C.isl_stream_close(s.e.h)
	for _, f := range s.free {
		f()
	}
	if rc != C.ISL_OK {
		return fmt.Errorf("isl_stream_close: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(s.e.h)))
	}
	return nil
}

// WhatIf runs `plan` against a device-side snapshot of the occupancy and puts the snapshot back: defragmentation planning
// ("would these pods fit if those slices were released?") without touching the live state (isl_snapshot_occupancy /
// isl_restore_occupancy: a 1-byte-per-GPU device copy).
func (e *PlacementEngine) WhatIf(plan func() error) error {
	if rc := C.isl_snapshot_occupancy(e.h); rc != C.ISL_OK {
		return fmt.Errorf("isl_snapshot_occupancy: %s", C.GoString(C.isl_strerror(rc)))
	}
	err := plan()
	if rc := C.isl_restore_occupancy(e.h); rc != C.ISL_OK && err == nil {
		err = fmt.Errorf("isl_restore_occupancy: %s", C.GoString(C.isl_strerror(rc)))
	}
	return err
}

// PreemptTarget is the answer of PreemptPending for one pod.  Victims empty and Placed: the pod fits as things are.  Not Placed: no GPU
// even with evictions.
type PreemptTarget struct {
	Placed   bool
	Nodename string
	GPUUUID  string
	Start    uint32
	Size     uint32
	Victims  []string // pod UIDs to delete before the pod is placed
}

// PreemptPending is priority preemption for the gated pods (ONE engine call, isl_preempt): for each pod, in order, the GPU and start it
// would take and the lower-priority pods that must leave first.  priority[i] is the PriorityClass value of pods[i]; podPriority maps the
// UID of each running pod to its value.  Values become dense order-preserving ranks (more than 255 distinct values is an error).  An
// Allocations entry is a victim only when its pod's priority is known, its status is not "deleted" and no other entry that marks slices
// busy (a dangling Prepared slice or another allocation) overlaps it; everything else is pinned.  Nothing is written to the custom
// resources: the caller deletes the victims, and once the daemonset has removed their allocations a later PlacePending places the pod.
func (r *InstasliceReconciler) PreemptPending(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, pods []PendingPod,
	priority []int32, podPriority map[string]int32) ([]PreemptTarget, error) {
	return r.preempt(e, list, pods, priority, podPriority, nil, nil)
}

// GangPreemptTarget is the answer of PreemptPendingGangs for one gang: Placed when every pod of the gang got a GPU, with one target per
// pod (their Victims empty) and the union of the pod UIDs to delete first.
type GangPreemptTarget struct {
	Placed  bool
	Pods    []PreemptTarget
	Victims []string
}

// PreemptPendingGangs is PreemptPending for gangs that must all run or none, ONE engine call on an engine created with FlagGangPreempt
// (include/islplace.h P1-P8): a gang gets victims for every pod or for none, a one-node gang goes to the node whose victims cost least.
// priority[k] is the PriorityClass value of every pod of gangs[k]; locality is nil, or one Gang* value per gang (any, one or distinct
// nodes) on an engine created with FlagGangLocality as well.  The caller deletes the union of the victims, then PlaceGangs places the
// gang once their allocations are gone; it fits there, though a greedy placement may choose other slices.
func (r *InstasliceReconciler) PreemptPendingGangs(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, gangs [][]PendingPod,
	priority []int32, podPriority map[string]int32, locality []uint8) ([]GangPreemptTarget, error) {
	if len(priority) != len(gangs) || (locality != nil && len(locality) != len(gangs)) {
		return nil, fmt.Errorf("one priority (and locality) per gang")
	}
	var pods []PendingPod
	var prio []int32
	var gangOf []uint32
	var loc []uint8
	for k, g := range gangs {
		if len(g) == 0 {
			return nil, fmt.Errorf("empty gang")
		}
		for _, p := range g {
			pods = append(pods, p)
			prio = append(prio, priority[k])
			gangOf = append(gangOf, uint32(k))
			if locality != nil {
				loc = append(loc, locality[k])
			}
		}
	}
	flat, err := r.preempt(e, list, pods, prio, podPriority, gangOf, loc)
	if err != nil {
		return nil, err
	}
	out := make([]GangPreemptTarget, len(gangs))
	i := 0
	for k, g := range gangs {
		t := GangPreemptTarget{Placed: true}
		seen := map[string]bool{}
		for j := range g {
			p := flat[i+j]
			t.Placed = t.Placed && p.Placed
			for _, v := range p.Victims {
				if !seen[v] {
					seen[v] = true
					t.Victims = append(t.Victims, v)
				}
			}
			p.Victims = nil
			t.Pods = append(t.Pods, p)
		}
		if !t.Placed {
			t = GangPreemptTarget{}
		}
		out[k] = t
		i += len(g)
	}
	return out, nil
}

// preempt is PreemptPending with, for gangs, a gang index per pod written into the request's handle and a locality byte into its start.
func (r *InstasliceReconciler) preempt(e *PlacementEngine, list *inferencev1alpha1.InstasliceList, pods []PendingPod, priority []int32,
	podPriority map[string]int32, gangOf []uint32, locality []uint8) ([]PreemptTarget, error) {
	out := make([]PreemptTarget, len(pods))
	if len(pods) == 0 {
		return out, nil
	}
	seen := map[int32]bool{}
	for _, v := range priority {
		seen[v] = true
	}
	for _, v := range podPriority {
		seen[v] = true
	}
	if len(seen) > 255 {
		return nil, fmt.Errorf("more than 255 distinct priority values")
	}
	values := make([]int32, 0, len(seen))
	for v := range seen {
		values = append(values, v)
	}
	sort.Slice(values, func(i, j int) bool { return values[i] < values[j] })
	rank := map[int32]uint8{}
	for i, v := range values {
		rank[v] = uint8(i)
	}
	span := func(start, size uint32) uint32 { return ((1 << size) - 1) << start }
	var victims []C.isl_victim
	var uids []string
	for g, uuid := range e.gpuUUID { // victims in (GPU, start) order
		spec := &list.Items[e.gpuNode[g]].Spec
		var masks []uint32 // every entry that marks slices of this GPU busy (:306-328)
		for _, p := range spec.Prepared {
			if p.Parent == uuid && p.PodUUID == "" {
				masks = append(masks, span(uint32(p.Start), uint32(p.Size)))
			}
		}
		var mine []string
		for uid, a := range spec.Allocations {
			if a.GPUUUID == uuid {
				masks = append(masks, span(uint32(a.Start), uint32(a.Size)))
				mine = append(mine, uid)
			}
		}
		sort.Slice(mine, func(i, j int) bool {
			ai, aj := spec.Allocations[mine[i]], spec.Allocations[mine[j]]
			return ai.Start < aj.Start || (ai.Start == aj.Start && mine[i] < mine[j])
		})
		for _, uid := range mine {
			a := spec.Allocations[uid]
			v, known := podPriority[uid]
			if !known || a.Allocationstatus == "deleted" {
				continue
			}
			m, overlapping := span(uint32(a.Start), uint32(a.Size)), 0
			for _, x := range masks {
				if x&m != 0 {
					overlapping++ // itself once; anything more would keep its slices busy
				}
			}
			if overlapping > 1 {
				continue
			}
			victims = append(victims, C.isl_victim{gpu: C.uint32_t(g), start: C.uint8_t(a.Start), size: C.uint8_t(a.Size), priority: C.uint8_t(rank[v])})
			uids = append(uids, uid)
		}
	}
	n := len(pods)
	reqP, resP := C.malloc(C.size_t(n)*C.sizeof_isl_request), C.malloc(C.size_t(n)*C.sizeof_isl_result)
	prioP, evictP := C.malloc(C.size_t(n)), C.malloc(C.size_t(n)*8*4)
	vicP := C.malloc(C.size_t(len(victims)+1) * C.sizeof_isl_victim)
	defer C.free(reqP)
	defer C.free(resP)
	defer C.free(prioP)
	defer C.free(evictP)
	defer C.free(vicP)
	if reqP == nil || resP == nil || prioP == nil || evictP == nil || vicP == nil {
		return nil, fmt.Errorf("out of memory")
	}
	req := (*[1 << 28]C.isl_request)(reqP)[:n:n]
	res := (*[1 << 28]C.isl_result)(resP)[:n:n]
	prio := (*[1 << 28]C.uint8_t)(prioP)[:n:n]
	evict := (*[1 << 28]C.uint32_t)(evictP)[: 8*n : 8*n]
	vic := (*[1 << 28]C.isl_victim)(vicP)[: len(victims)+1 : len(victims)+1]
	copy(vic, victims)
	e.fillRequests(req, pods, 0)
	for i := range pods {
		prio[i] = C.uint8_t(rank[priority[i]])
		if gangOf != nil {
			req[i].handle = C.uint32_t(gangOf[i])
		}
		if locality != nil {
			req[i].start = C.uint8_t(locality[i])
		}
	}
	if rc := C.isl_preempt(e.h, C.uint32_t(n), &req[0], &prio[0], C.uint32_t(len(victims)), &vic[0], &res[0], &evict[0]); rc != C.ISL_OK {
		return nil, fmt.Errorf("isl_preempt: %s (%s)", C.GoString(C.isl_strerror(rc)), C.GoString(C.isl_last_cuda_error(e.h)))
	}
	for i := range pods {
		if res[i].status != C.ISL_ST_PLACED {
			continue
		}
		g := int(res[i].gpu)
		t := PreemptTarget{Placed: true, Nodename: list.Items[e.gpuNode[g]].Name, GPUUUID: e.gpuUUID[g],
			Start: uint32(res[i].start), Size: uint32(res[i].size)}
		for k := 0; k < 8; k++ {
			if idx := uint32(evict[8*i+k]); idx != C.ISL_GPU_NONE {
				t.Victims = append(t.Victims, uids[idx])
			}
		}
		out[i] = t
	}
	return out, nil
}
