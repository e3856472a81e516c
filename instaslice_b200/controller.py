"""Host-side mirror of the reference's allocator interface, backed by the CUDA engine.

The reference's controller is Go and Go cannot be compiled in this image, so this module plays the part of
the Go shim described in INTEGRATION.md: same names, argument meaning and error behaviour as
``internal/controller/instaslice_controller.go`` for the allocator path, on CR-shaped dicts (JSON field names of
``api/v1alpha1/instaslice_types.go``).  Nothing here decides a placement: occupancy bytes and profile rows are
*derived* from the custom resources exactly the way the reference reads them, and every decision comes back
from ``libislplace.so`` through the C ABI.

  InstasliceReconciler.findDeviceForASlice            :240-262
  InstasliceReconciler.getStartIndexFromPreparedState :303-384   (occupancy build :306-328 is ``occupancy_byte``)
  InstasliceReconciler.extractGpuProfile              :283-300
  InstasliceReconciler.extractProfileName             :265-280
  FirstFitPolicy.SetAllocationDetails                 :436-453
  InstasliceReconciler.reconcile_gated_pod            the node loop + Prepared veto of Reconcile :188-232
  InstasliceReconciler.place_pending_pods             the batched entry the engine was built for
"""
from __future__ import annotations

import re

import numpy as np

from . import engine as E

NOT_VALID_INDEX = 9   # :248, :343
ERR_NO_GPU = "failed to find allocatable gpu"   # :261


class AllocationError(Exception):
    """The Go ``error`` value of findDeviceForASlice."""


class FirstFitPolicy:
    """:436-453 — packs the twelve arguments into AllocationDetails; it chooses nothing."""

    def SetAllocationDetails(self, profileName, newStart, size, podUUID, nodename, processed, discoveredGiprofile,
                             Ciprofileid, Ciengprofileid, namespace, podName, gpuUuid):
        return {"profile": profileName, "start": int(newStart), "size": int(size), "podUUID": podUUID, "gpuUUID": gpuUuid,
                "nodename": nodename, "allocationStatus": processed, "giprofileid": discoveredGiprofile,
                "ciProfileid": Ciprofileid, "ciengprofileid": Ciengprofileid, "namespace": namespace, "podName": podName}


class LeftToRightPolicy:
    """:456-461 — a stub in the reference: returns an empty AllocationDetails."""

    def SetAllocationDetails(self, *args):
        return {}


class RightToLeftPolicy(LeftToRightPolicy):
    """:464-469 — same stub."""


def occupancy_byte(instaslice: dict, gpu_uuid: str) -> int:
    """:306-328 — dangling Prepared (PodUUID == "") and every Allocations entry (any status) mark their slices."""
    spec = instaslice["spec"]
    busy = 0
    for item in spec.get("prepared", {}).values():
        if item["parent"] == gpu_uuid and item.get("podUUID", "") == "":
            if item["start"] + item["size"] > 8:
                raise ValueError("prepared span beyond slice 7 (the reference would panic, :316)")
            busy |= ((1 << int(item["size"])) - 1) << int(item["start"])
    for item in spec.get("allocations", {}).values():
        if item["gpuUUID"] == gpu_uuid:
            if item["start"] + item["size"] > 8:
                raise ValueError("allocation span beyond slice 7 (the reference would panic, :325)")
            busy |= ((1 << int(item["size"])) - 1) << int(item["start"])
    return busy & 0xFF


def profile_rows(migplacement: list):
    """``spec.migplacement`` -> (isl_profile records, {name: row index}).

    The start search uses the FIRST row with a given name (:332-340, ``break``); row order is kept so that
    index == position of that first row.  Duplicate starts inside a row are dropped (they cannot change the
    first hit).  A row with an empty placement list makes the reference panic (:334): rejected here.
    """
    names, table = {}, []
    for row in migplacement:
        if row["profile"] in names:
            continue
        if not row.get("placements"):
            raise ValueError("Migplacement row %r has no placements (reference panics at :334)" % row["profile"])
        names[row["profile"]] = len(table)
        table.append((row["profile"], row["placements"][0]["size"], [p["start"] for p in row["placements"]], row["giprofileid"]))
    if len(table) > E.MAX_PROFILES:
        raise ValueError("more than %d distinct profiles" % E.MAX_PROFILES)
    return E.make_profiles(table), names


class InstasliceReconciler:
    """Allocator half of the reference's ``InstasliceReconciler`` over a list of Instaslice objects.

    The engine mirrors the listed custom resources (``sync``); GPUs are in canonical order: nodes in list order,
    GPUs by ascending UUID inside a node (the reference's orders are random, SURVEY Q6).
    """

    def __init__(self, instaslices: list, quirks: int = E.QUIRKS_REF_EXACT, max_batch: int = 65536, engine: E.Engine | None = None,
                 policy: int = E.POLICY_FIRST_FIT, gang_one_node: bool = False, gang_distinct_nodes: bool = False,
                 gang_few_nodes: bool = False, gang_locality: bool = False, gang_min_members: bool = False, gang_preempt: bool = False,
                 gang_node_score: bool = False, gang_balanced: bool = False, gang_node_score_all: bool = False,
                 first_available: bool = False):
        """``policy``: the engine policy of the engine this reconciler creates (``engine`` is None), e.g. ``E.POLICY_MOST_ALLOCATED`` to
        pack MIG pods onto the fullest nodes or ``E.POLICY_LEAST_ALLOCATED`` to spread them (include/islplace.h).  ``gang_one_node``:
        that engine is created with ``E.FLAG_GANG_ONE_NODE``, so ``place_pending_gangs`` puts every gang on one node.
        ``gang_distinct_nodes``: with ``E.FLAG_GANG_DISTINCT_NODES``, so it puts every member of a gang on a different node (the engine
        refuses both flags at once).  ``gang_few_nodes``: with ``E.FLAG_GANG_FEW_NODES``, so it puts a gang on one node when one takes
        it, else on as few nodes as it greedily can (the engine refuses it with either of the other two).  ``gang_locality``: with
        ``E.FLAG_GANG_LOCALITY``, so ``place_pending_gangs`` takes a locality per gang (the engine refuses it with the other three).
        ``gang_min_members``: with ``E.FLAG_GANG_MIN_MEMBERS`` (alone or with one of the four), so ``place_pending_gangs`` takes a
        minimum per gang and may place a gang's leading pods only.  ``gang_preempt``: with ``E.FLAG_GANG_PREEMPT`` (alone or with the
        one-node, distinct-node or locality flag), so ``preempt_pending_gangs`` picks the victims of whole gangs.  ``gang_node_score``:
        with ``E.FLAG_GANG_NODE_SCORE``, for a ``POLICY_MOST_ALLOCATED`` or ``POLICY_LEAST_ALLOCATED`` reconciler, so that
        ``place_pending_gangs`` places gangs by the node score, alone (any node) or with the one-node, distinct-node or locality option
        (the engine refuses it with any other policy, few-node gangs and elastic gangs).  ``gang_balanced``: with
        ``E.FLAG_GANG_BALANCED``, which needs ``gang_locality``, so that a gang's locality may be ``E.gang_balanced_nodes(k)``: its
        replicas spread over the nodes within a maxSkew of k (the engine refuses it under node scoring unless ``gang_node_score_all``).
        ``gang_node_score_all``: with ``E.FLAG_GANG_NODE_SCORE_ALL``, which needs ``gang_node_score``, so that the node score also places
        few-node gangs (``gang_few_nodes`` or a ``GANG_FEW_NODES`` locality), elastic gangs (``gang_min_members``) and balanced gangs
        (``gang_balanced``), all on the one packing or spreading engine.  ``first_available``: with ``E.FLAG_FIRST_AVAILABLE``, so that a
        pod given to ``place_pending_pods`` may list ``"fallbacks"``, profiles it also accepts, and gets the first of its profiles that
        fits (include/islplace.h A1-A8)."""
        self.quirks = quirks
        self.policy = policy
        self.gang_one_node = gang_one_node
        self.gang_distinct_nodes = gang_distinct_nodes
        self.gang_few_nodes = gang_few_nodes
        self.gang_locality = gang_locality
        self.gang_min_members = gang_min_members
        self.gang_preempt = gang_preempt
        self.gang_node_score = gang_node_score
        self.gang_balanced = gang_balanced
        self.gang_node_score_all = gang_node_score_all
        self.first_available = first_available
        self.items = instaslices
        self._engine = engine
        self._max_batch = max_batch
        self.sync()

    # -- CR -> engine ---------------------------------------------------------------------------
    def sync(self):
        """Rebuild the flat inventory from the custom resources (the CR is the checkpoint)."""
        if not self.items:
            raise ValueError("no Instaslice objects")
        # every node publishes its own Migplacement (instaslice_daemonset.go:588-664): group identical tables
        self._tables, self.node_table = [], []
        for it in self.items:
            mig = it["spec"].get("migplacement", [])
            if mig not in self._tables:
                if len(self._tables) >= 8:
                    raise ValueError("more than 8 distinct per-node profile tables")
                self._tables.append(mig)
            self.node_table.append(self._tables.index(mig))
        per_table = [profile_rows(mig) for mig in self._tables]
        self.profile_names = {}
        for _rows, names in per_table:                       # profile NAME index = order of first appearance over the tables
            for name in names:
                self.profile_names.setdefault(name, len(self.profile_names))
        if len(self.profile_names) > E.MAX_PROFILES:
            raise ValueError("more than %d distinct profile names" % E.MAX_PROFILES)
        self.rows = np.zeros((len(self._tables), len(self.profile_names)), dtype=E.PROFILE_DTYPE)
        for t, (rows, names) in enumerate(per_table):
            for name, idx in names.items():
                self.rows[t, self.profile_names[name]] = rows[idx]
        self.gpu_uuid, node_off, occ = [], [0], []
        self.node_of_uuid = {}
        for n, it in enumerate(self.items):
            for uuid in sorted(it["spec"].get("MigGPUUUID", {})):
                self.gpu_uuid.append(uuid)
                self.node_of_uuid[uuid] = n
                occ.append(occupancy_byte(it, uuid))
            node_off.append(len(self.gpu_uuid))
        self.node_off = np.asarray(node_off, dtype=np.uint32)
        self.gpu_index = {u: i for i, u in enumerate(self.gpu_uuid)}
        if self._engine is None:
            self._engine = E.Engine(max_gpus=max(4096, len(self.gpu_uuid)), max_batch=self._max_batch, policy=self.policy, quirks=self.quirks,
                                    flags=(E.FLAG_GANG_ONE_NODE if self.gang_one_node else 0) |
                                          (E.FLAG_GANG_DISTINCT_NODES if self.gang_distinct_nodes else 0) |
                                          (E.FLAG_GANG_FEW_NODES if self.gang_few_nodes else 0) |
                                          (E.FLAG_GANG_LOCALITY if self.gang_locality else 0) |
                                          (E.FLAG_GANG_MIN_MEMBERS if self.gang_min_members else 0) |
                                          (E.FLAG_GANG_PREEMPT if self.gang_preempt else 0) |
                                          (E.FLAG_GANG_NODE_SCORE if self.gang_node_score else 0) |
                                          (E.FLAG_GANG_BALANCED if self.gang_balanced else 0) |
                                          (E.FLAG_GANG_NODE_SCORE_ALL if self.gang_node_score_all else 0) |
                                          (E.FLAG_FIRST_AVAILABLE if self.first_available else 0))
        self._engine.load_profile_tables(self.rows)
        self._engine.load_inventory(self.node_off, np.asarray(occ, dtype=np.uint8))
        self._engine.set_node_tables(np.asarray(self.node_table, dtype=np.uint8))
        # spans of realised slices whose Allocations entry is gone: only these can trigger the veto (:198-203)
        self._has_orphans = any(
            p.get("podUUID", "") != "" and p["podUUID"] not in it["spec"].get("allocations", {})
            for it in self.items for p in it["spec"].get("prepared", {}).values())

    def update_node(self, instaslice: dict):
        """Incremental sync after ONE Instaslice object changed (an Allocations / Prepared entry appeared, changed or was
        deleted by the daemonset): recompute the occupancy bytes of that node's GPUs only and overwrite them in the engine.
        Falls back to a full ``sync`` when the node's GPU set or profile table changed."""
        n = next((i for i, it in enumerate(self.items) if it["metadata"]["name"] == instaslice["metadata"]["name"]), None)
        if n is None:
            self.items.append(instaslice)
            return self.sync()
        lo, hi = int(self.node_off[n]), int(self.node_off[n + 1])
        uuids = sorted(instaslice["spec"].get("MigGPUUUID", {}))
        if uuids != self.gpu_uuid[lo:hi] or instaslice["spec"].get("migplacement", []) != self._tables[self.node_table[n]]:
            self.items[n] = instaslice
            return self.sync()
        self.items[n] = instaslice
        self._engine.write_occupancy(lo, np.array([occupancy_byte(instaslice, u) for u in uuids], dtype=np.uint8))
        self._has_orphans = any(
            p.get("podUUID", "") != "" and p["podUUID"] not in it["spec"].get("allocations", {})
            for it in self.items for p in it["spec"].get("prepared", {}).values())

    @property
    def engine(self) -> E.Engine:
        return self._engine

    # -- reference-named helpers ----------------------------------------------------------------
    @staticmethod
    def extractProfileName(limits: dict) -> str:
        """:265-280"""
        name = ""
        for k in sorted(limits):
            if "nvidia" in k:
                m = re.search(r"(\d+g\.\d+gb)", k)
                if m:
                    name = m.group(1)
        return name

    @staticmethod
    def extractGpuProfile(instaslice: dict, profileName: str):
        """:283-300 — the LAST matching row wins; size of its first placement."""
        size = gi = ci = cieng = 0
        for row in instaslice["spec"].get("migplacement", []):
            if row["profile"] == profileName:
                for p in row.get("placements", []):
                    size, gi, ci, cieng = p["size"], row["giprofileid"], row["ciProfileid"], row["ciengprofileid"]
                    break
        return size, gi, ci, cieng

    def getStartIndexFromPreparedState(self, instaslice: dict, gpuUUID: str, profileName: str) -> int:
        """:303-384 — the occupancy byte comes from the CR, the search from the device table."""
        row = self.profile_names.get(profileName)
        if row is None:
            return NOT_VALID_INDEX
        occ = np.array([occupancy_byte(instaslice, gpuUUID)], dtype=np.uint8)
        n = next(i for i, it in enumerate(self.items) if it is instaslice or it["metadata"]["name"] == instaslice["metadata"]["name"])
        return int(self._engine.eval_starts(row | (self.node_table[n] << 8), occ)[0])       # the node's own table

    def findDeviceForASlice(self, instaslice: dict, profileName: str, policy, pod: dict) -> dict:
        """:240-262 — first GPU of ONE node with a valid start; raises AllocationError(:261) when none.

        Like the reference this does not write the allocation into the CR (:257 is commented out there); the engine's
        occupancy is left untouched as well (the tentative commit is released again).
        """
        n = next(i for i, it in enumerate(self.items) if it is instaslice)
        lo, hi = int(self.node_off[n]), int(self.node_off[n + 1])
        res = self._place([profileName], lo, hi)[0]
        if res["status"] != E.ST_PLACED:
            raise AllocationError(ERR_NO_GPU)
        self._release(res)
        return self._details(instaslice, profileName, policy, pod, res)

    # -- Reconcile's node loop, one pod (:188-232) ------------------------------------------------
    def reconcile_gated_pod(self, pod: dict, profileName: str, policy=None):
        """Returns ("placed", AllocationDetails) | ("veto", None) | ("none", None); on "placed" the allocation is
        written to the owning Instaslice (``r.Update``, :218-219).  Canonical semantics: the first node with
        capacity wins (the reference has no ``break`` there, SURVEY Q5)."""
        policy = policy or FirstFitPolicy()
        res = self._place([profileName], 0, len(self.gpu_uuid))[0]
        if res["status"] != E.ST_PLACED:
            return ("none", None)
        return self._commit_or_veto(pod, profileName, policy, res)

    # -- the batched entry ------------------------------------------------------------------------
    def place_pending_pods(self, pods: list, policy=None):
        """Resolve many gated pods ``[{"uid","name","namespace","profile"}]`` in order with ONE engine call.

        Returns a list of ("placed", AllocationDetails) | ("veto", None) | ("none", None).  When the cluster holds
        realised slices whose allocation is already gone (the only state in which the reference's exact-match veto
        can fire) the pods are resolved one engine call each, so that a vetoed pod leaves no trace before the next
        one is looked at — exactly the reference's sequence.

        On a ``first_available`` reconciler a pod may carry ``"fallbacks": [names...]``, profiles it also accepts, in order of
        preference after ``"profile"``.  The pod's names become one run of requests with the pod's index as handle, and the pod gets the
        first of them that fits when its turn comes (include/islplace.h A1-A8).  Its AllocationDetails name the chosen profile: its
        ``profile``, ``size`` and GI / CI ids come from ``extractGpuProfile`` of that name, so the daemonset creates that slice.  The
        veto applies to the chosen span as to any other pod's.  A pod with fallbacks on any other reconciler raises ``ValueError``.
        """
        policy = policy or FirstFitPolicy()
        names = [self._alternatives(p) for p in pods]
        if self._has_orphans:
            return [self._reconcile_alternatives(p, alts, policy) for p, alts in zip(pods, names)]
        out = []
        handles = [i for i, alts in enumerate(names) for _ in alts]
        results = self._place([n for alts in names for n in alts], 0, len(self.gpu_uuid), handles)
        k = 0
        for pod, alts in zip(pods, names):
            out.append(self._chosen(pod, alts, results[k:k + len(alts)], policy))
            k += len(alts)
        return out

    def _alternatives(self, pod: dict) -> list:
        """A pending pod's profile names in order of preference: its profile, then its fallbacks (``first_available`` only)."""
        fallbacks = list(pod.get("fallbacks") or [])
        if fallbacks and not self.first_available:
            raise ValueError("a pod with fallbacks needs a reconciler created with first_available=True")
        return [pod["profile"], *fallbacks]

    def _chosen(self, pod, alts, res, policy):
        """The outcome of one pod from the records of its alternatives: the PLACED one, if any, names the profile."""
        for name, r in zip(alts, res):
            if r["status"] == E.ST_PLACED:
                return self._commit_or_veto(pod, name, policy, r)
        return ("none", None)

    def _reconcile_alternatives(self, pod, alts, policy):
        """reconcile_gated_pod for a pod's whole run of alternatives: one engine call."""
        if len(alts) == 1:
            return self.reconcile_gated_pod(pod, alts[0], policy)
        return self._chosen(pod, alts, self._place(alts, 0, len(self.gpu_uuid), [0] * len(alts)), policy)

    def place_pending_gangs(self, gangs: list, policy=None, locality=None, min_members=None):
        """All-or-nothing pod groups (the replicas of one deployment, the workers of one job): ``gangs`` is a list of non-empty pod
        lists shaped as ``place_pending_pods`` takes them, resolved in order with ONE engine call (isl_place_gangs).

        Returns per gang ("placed", [AllocationDetails...]) | ("veto", None) | ("none", None).  A gang is placed only when every pod of
        it gets a slice, and only then are its allocations written to the custom resources.  When the Prepared exact-match veto
        (:198-203) fires on any pod, the spans of the whole gang are released again.  With realised slices whose allocation is gone
        (the only state in which the veto can fire) the gangs are resolved one engine call each, as ``place_pending_pods`` does per pod.

        ``locality``: one ``E.GANG_*`` value per gang (e.g. from Kueue's podset topology annotations, INTEGRATION.md), for a reconciler
        created with ``gang_locality=True``: a training job on one node, replicas on distinct nodes, a job on few nodes and free pods in
        one call on one occupancy.  With ``gang_balanced=True`` as well, ``E.gang_balanced_nodes(k)`` spreads a Deployment's replicas
        over the nodes within a maxSkew of k (``topologySpreadConstraints`` on ``kubernetes.io/hostname``), more replicas than nodes
        included.

        ``min_members``: one minimum m (0..255) per gang (the PodGroup's minMember, Volcano's minAvailable or Kueue's PodSet minCount,
        INTEGRATION.md), for a reconciler created with ``gang_min_members=True``.  A gang whose leading pods reach its minimum while a
        later pod finds no slice is placed with those pods only: its allocation list is shorter than the gang, and only those pods'
        allocations are written.  List the pods the job needs first: the placed pods are always a leading run.
        """
        policy = policy or FirstFitPolicy()
        if any(not g for g in gangs):
            raise ValueError("empty gang")
        if self._has_orphans and len(gangs) > 1:
            locs = [None] * len(gangs) if locality is None else [[loc] for loc in locality]
            mins = [None] * len(gangs) if min_members is None else [[m] for m in min_members]
            return [self.place_pending_gangs([g], policy, loc, m)[0] for g, loc, m in zip(gangs, locs, mins)]
        if not gangs:
            return []
        off = np.cumsum([0] + [len(g) for g in gangs]).astype(np.uint32)
        results = self._engine.place_gangs(self._requests([p["profile"] for g in gangs for p in g]), off, locality, min_members)
        out = []
        for gang, a, b in zip(gangs, off[:-1], off[1:]):
            placed = int((results["status"][a:b] == E.ST_PLACED).sum())    # a leading run: all, none, or an elastic gang's first pods
            if placed == 0:
                out.append(("none", None))
                continue
            gang, res = gang[:placed], results[a:a + placed]
            packed = [self._alloc_for(pod, pod["profile"], policy, r) for pod, r in zip(gang, res)]
            if any(self._vetoed(instaslice, alloc) for instaslice, alloc in packed):
                spans = np.zeros(len(res), dtype=E.SPAN_DTYPE)
                spans["gpu"], spans["start"], spans["size"] = res["gpu"], res["start"], res["size"]
                self._engine.free_batch(spans)
                out.append(("veto", None))
                continue
            for pod, (instaslice, alloc) in zip(gang, packed):
                instaslice["spec"].setdefault("allocations", {})[pod["uid"]] = alloc   # :215-219
            out.append(("placed", [alloc for _, alloc in packed]))
        return out

    def preempt_pending_pods(self, pods: list, pod_priority: dict):
        """Priority preemption for gated pods the kube-scheduler never sees as MIG-constrained (ONE engine call, isl_preempt).

        ``pods`` are shaped as ``place_pending_pods`` takes them, each with a ``"priority"`` (the int32 value of its PriorityClass);
        ``pod_priority`` maps the UID of each running pod to its value.  Values become dense order-preserving ranks over every value
        seen (more than 255 distinct values is a ``ValueError``).  An ``Allocations`` entry may be evicted only when its pod's priority
        is known, its status is not ``"deleted"`` (it is already leaving) and no other entry that marks slices busy (a dangling
        Prepared slice or another allocation) overlaps its span, for otherwise releasing it would not free its slices; every other
        busy slice is pinned.

        Returns per pod ("fits", None, []) | ("preempt", {"nodename", "gpuUUID", "start", "size"}, [victim pod UIDs]) |
        ("none", None, []).  Nothing is written to the custom resources: the caller deletes the victim pods, and once the daemonset
        has removed their allocations a later ``place_pending_pods`` places the pod on the reported slices (first-fit engine).
        """
        rank, victims, uids = self._victims(pods, pod_priority)
        res, evict = self._engine.preempt(self._requests([p["profile"] for p in pods]),
                                          np.array([rank[int(p["priority"])] for p in pods], dtype=np.uint8), victims)
        out = []
        for r, row in zip(res, evict):
            if r["status"] != E.ST_PLACED:
                out.append(("none", None, []))
                continue
            gone = [uids[int(k)] for k in row if k != E.GPU_NONE]
            out.append(("preempt", self._where(r), gone) if gone else ("fits", None, []))
        return out

    def preempt_pending_gangs(self, gangs: list, pod_priority: dict, locality=None):
        """Gang preemption (ONE engine call, isl_preempt on an engine created with ``gang_preempt=True``): for each gang of pods that
        must all run or none, the slices its pods would take and the running pods that must leave first, or nothing when the gang
        cannot run even then.  ``gangs`` are lists of pods shaped as ``preempt_pending_pods`` takes them; the pods of one gang carry one
        priority (else ``ValueError``).  The victims may be any ``Allocations`` entry ``preempt_pending_pods`` may evict.
        ``locality``: one ``E.GANG_*`` value per gang (0, 1 or 3) for a reconciler created with ``gang_locality=True`` as well.

        Returns per gang ("fits", None, []) | ("preempt", [{"nodename", "gpuUUID", "start", "size"} per pod], [victim pod UIDs]) |
        ("none", None, []).  Nothing is written to the custom resources: the caller deletes the union of the victims, and once their
        allocations are gone ``place_pending_gangs`` places the gang (include/islplace.h P6 (d): it fits where it was shown, though a
        greedy placement may choose other slices).
        """
        if any(not g for g in gangs):
            raise ValueError("empty gang")
        if any(len({int(p["priority"]) for p in g}) > 1 for g in gangs):
            raise ValueError("the pods of one gang have different priorities")
        if not gangs:
            return []
        pods = [p for g in gangs for p in g]
        rank, victims, uids = self._victims(pods, pod_priority)
        off = np.cumsum([0] + [len(g) for g in gangs])
        res, evict = self._engine.preempt(self._requests([p["profile"] for p in pods]),
                                          np.array([rank[int(p["priority"])] for p in pods], dtype=np.uint8), victims, off, locality)
        out = []
        for a, b in zip(off[:-1], off[1:]):
            if (res["status"][a:b] != E.ST_PLACED).any():
                out.append(("none", None, []))
                continue
            gone = sorted({int(k) for row in evict[a:b] for k in row if k != E.GPU_NONE})
            out.append(("preempt", [self._where(r) for r in res[a:b]], [uids[k] for k in gone]) if gone else ("fits", None, []))
        return out

    def _victims(self, pods, pod_priority):
        """Dense priority ranks over every value seen, the victims (VICTIM_DTYPE) and their pod UIDs (preempt_pending_pods)."""
        values = sorted({int(p["priority"]) for p in pods} | {int(v) for v in pod_priority.values()})
        if len(values) > 255:
            raise ValueError("more than 255 distinct priority values")
        rank = {v: r for r, v in enumerate(values)}
        victims, uids = [], []
        for n, it in enumerate(self.items):
            spec = it["spec"]
            for g in range(int(self.node_off[n]), int(self.node_off[n + 1])):
                uuid = self.gpu_uuid[g]
                entries = [(None, p) for p in spec.get("prepared", {}).values() if p["parent"] == uuid and p.get("podUUID", "") == ""]
                entries += [(uid, a) for uid, a in spec.get("allocations", {}).items() if a["gpuUUID"] == uuid]
                masks = [((1 << int(x["size"])) - 1) << int(x["start"]) for _, x in entries]
                for j, (uid, a) in sorted(enumerate(entries), key=lambda e: int(e[1][1]["start"])):
                    if uid is None or uid not in pod_priority or a.get("allocationStatus") == "deleted":
                        continue
                    if any(masks[j] & m for k, m in enumerate(masks) if k != j):
                        continue
                    victims.append((g, int(a["start"]), int(a["size"]), rank[int(pod_priority[uid])], 0))
                    uids.append(uid)
        return rank, np.array(victims, dtype=E.VICTIM_DTYPE), uids

    def _where(self, r):
        uuid = self.gpu_uuid[int(r["gpu"])]
        return {"nodename": self.items[self.node_of_uuid[uuid]]["metadata"]["name"], "gpuUUID": uuid, "start": int(r["start"]),
                "size": int(r["size"])}

    def release(self, pod_uid: str):
        """The daemonset deleted ``Allocations[podUID]`` (instaslice_daemonset.go:261-263): free its span."""
        for n, it in enumerate(self.items):
            a = it["spec"].get("allocations", {}).pop(pod_uid, None)
            if a is not None:
                # rebuild the node's bytes from the CR (OR over every remaining entry, :306-328) instead of clearing the span blindly:
                # slices another entry still covers stay busy, exactly what the reference's next rebuild would say
                lo, hi = int(self.node_off[n]), int(self.node_off[n + 1])
                self._engine.write_occupancy(lo, np.array([occupancy_byte(it, u) for u in self.gpu_uuid[lo:hi]], dtype=np.uint8))
                return True
        return False

    # -- internals --------------------------------------------------------------------------------
    def _requests(self, profile_names, handles=None):
        req = np.zeros(len(profile_names), dtype=E.REQUEST_DTYPE)
        req["handle"] = np.arange(len(profile_names), dtype=np.uint32) if handles is None else np.asarray(handles, dtype=np.uint32)
        req["profile"] = [self.profile_names.get(n, E.PROFILE_UNKNOWN) for n in profile_names]
        req["op"] = E.OP_ALLOC
        return req

    def _place(self, profile_names, lo, hi, handles=None):
        # ONE locked call restricts, places and restores (isl_place_batch_range): two reconcile workers cannot interleave and
        # nothing leaks when the call fails
        return self._engine.place_batch_range(lo, hi, self._requests(profile_names, handles))

    def _release(self, res):
        spans = np.zeros(1, dtype=E.SPAN_DTYPE)
        spans[0] = (res["gpu"], res["start"], res["size"], 0)
        self._engine.free_batch(spans)

    def _details(self, instaslice, profileName, policy, pod, res):
        size, gi, ci, cieng = self.extractGpuProfile(instaslice, profileName)
        return policy.SetAllocationDetails(profileName, int(res["start"]), size, pod["uid"], instaslice["metadata"]["name"],
                                           "creating", gi, ci, cieng, pod.get("namespace", "default"), pod["name"],
                                           self.gpu_uuid[int(res["gpu"])])

    def _alloc_for(self, pod, profileName, policy, res):
        """The owning Instaslice of a PLACED record and the AllocationDetails the policy packs for it."""
        instaslice = self.items[self.node_of_uuid[self.gpu_uuid[int(res["gpu"])]]]
        return instaslice, self._details(instaslice, profileName, policy, pod, res)

    @staticmethod
    def _vetoed(instaslice, alloc):
        return any(item["parent"] == alloc["gpuUUID"] and item["size"] == alloc["size"] and item["start"] == alloc["start"]
                   for item in instaslice["spec"].get("prepared", {}).values())          # :198-203

    def _commit_or_veto(self, pod, profileName, policy, res):
        instaslice, alloc = self._alloc_for(pod, profileName, policy, res)
        if self._vetoed(instaslice, alloc):
            self._release(res)
            return ("veto", None)
        instaslice["spec"].setdefault("allocations", {})[pod["uid"]] = alloc   # :215-219
        return ("placed", alloc)
