"""CPU restatements of isl_place_gangs (TEST INFRASTRUCTURE, NOT PRODUCT CODE): the checkers of the gang tests and of
tools/gang_time.py.

``fast_place_gangs``  the gang rules of include/islplace.h over ``oracle.Fast`` (ref_fast.cpp), which places one request after the
                      other under every policy: each gang's ALLOCs go through one ``place`` call; when one of them is not PLACED the
                      spans the call did place are released again with FREE requests (disjoint spans that were free before, so the
                      occupancy and ref_fast's per-profile cursors are exactly those of the gang's start).
``ref_py_place_gangs`` first-fit on CR-shaped dicts: ``ref_py.reconcile_gated_pod`` member by member on a deep copy of the custom
                      resources, and the copy is kept or dropped.  Shares nothing with the first beyond the rules.
"""
from __future__ import annotations

import copy

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import alloc_requests
from oracle import ref_py

# The known-answer vector, derived by hand from the rules: one node with one empty A100-40GB GPU, reference-exact quirks, first-fit.
# Gang 2 sees 3g.20gb alive again after it "died" inside the aborted gang 1.
A100 = {name: i for i, (name, *_rest) in enumerate(tables.A100_40GB)}
_NONE, _ABORTED, _NO_CAP, _PLACED = E.GPU_NONE, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_PLACED
KAT_GANGS = [["3g.20gb", "3g.20gb"], ["3g.20gb", "1g.5gb"], ["1g.5gb", "2g.10gb"], ["1g.5gb", "1g.5gb"], ["1g.5gb"]]
KAT_RECORDS = [[(_NONE, 9, 4, _ABORTED), (_NONE, 9, 4, _NO_CAP)], [(0, 0, 4, _PLACED), (0, 4, 1, _PLACED)],
               [(_NONE, 9, 1, _ABORTED), (_NONE, 9, 2, _NO_CAP)], [(0, 5, 1, _PLACED), (0, 6, 1, _PLACED)], [(_NONE, 9, 1, _NO_CAP)]]
KAT_OCC = [0x00, 0x1F, 0x1F, 0x7F, 0x7F]     # occupancy byte after each gang


def kat_call():
    """The known-answer gangs as one call: requests and gang offsets."""
    names = [n for g in KAT_GANGS for n in g]
    req = alloc_requests(np.array([A100[n] for n in names], dtype=np.uint8))
    return req, np.cumsum([0] + [len(g) for g in KAT_GANGS]).astype(np.uint32)


def default_sizes(rows, node_table=None) -> list:
    """Size an unplaced ALLOC of each profile reports: its row in the table of the first node (canonical order) that has one, else 0."""
    rows = np.asarray(rows)
    if rows.ndim == 1:
        return [int(r["size"]) for r in rows]
    out = []
    for p in range(rows.shape[1]):
        t = next((int(t) for t in node_table if rows[int(t), p]["n_starts"]), None)
        out.append(int(rows[t, p]["size"]) if t is not None else 0)
    return out


def fast_place_gangs(ref, requests, gang_off, sizes) -> np.ndarray:
    """``ref``: an ``oracle.Fast`` holding the occupancy; ``sizes``: ``default_sizes`` of its tables.  Returns the records of
    isl_place_gangs and leaves the final occupancy in ``ref``."""
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.asarray(gang_off, dtype=np.int64)
    alloc = req["op"] == E.OP_ALLOC
    frees = req.copy()
    frees["op"][alloc] = E.OP_NOOP
    out = ref.place(frees)                      # every FREE of the call first; NOOP records for the rest
    for a, b in zip(gang_off[:-1], gang_off[1:]):
        idx = np.flatnonzero(alloc[a:b]) + a
        if len(idx) == 0:
            continue
        res = ref.place(req[idx])
        failed = np.flatnonzero(res["status"] != E.ST_PLACED)
        if len(failed) == 0:
            out[idx] = res
            continue
        done = res[res["status"] == E.ST_PLACED]
        undo = np.zeros(len(done), dtype=E.REQUEST_DTYPE)
        undo["handle"], undo["op"], undo["start"], undo["size"] = done["gpu"], E.OP_FREE, done["start"], done["size"]
        ref.place(undo)
        for i in idx:
            p = int(req["profile"][i])
            out[i] = (E.GPU_NONE, E.START_NONE, sizes[p] if p < len(sizes) else 0, E.ST_GANG_ABORTED)
        out[idx[failed[0]]] = res[failed[0]]
    return out


def cluster_crs(node_off, node_table, occ, table_list) -> list:
    """One Instaslice dict per node; GPU g is "GPU-%012d" % g (canonical = ascending UUID), busy slices as dangling Prepared."""
    crs = []
    for n in range(len(node_off) - 1):
        spec = {"MigGPUUUID": {}, "allocations": {}, "prepared": {}, "migplacement": tables.migplacement(table_list[int(node_table[n])])}
        for g in range(int(node_off[n]), int(node_off[n + 1])):
            uuid = "GPU-%012d" % g
            spec["MigGPUUUID"][uuid] = "x"
            for s in range(8):
                if (int(occ[g]) >> s) & 1:
                    spec["prepared"]["MIG-%d-%d" % (g, s)] = {"profile": "", "start": s, "size": 1, "parent": uuid, "podUUID": "",
                                                              "giinfo": 0, "ciinfo": 0}
        crs.append({"metadata": {"name": "node-%03d" % n}, "spec": spec})
    return crs


def ref_py_place_gangs(crs: list, gangs: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``.  First-fit, the reference's node loop per member on a deep copy of ``crs``; a gang
    whose members all come back "placed" replaces ``crs``' contents with the copy.  Returns per gang ("placed", [AllocationDetails...])
    or ("aborted", index of the member that found nothing)."""
    out = []
    for gang in gangs:
        shadow = copy.deepcopy(crs)
        allocs = []
        for k, (pod, name) in enumerate(gang):
            verdict, placed = ref_py.reconcile_gated_pod(shadow, pod, name, quirks)
            if verdict != "placed":
                out.append(("aborted", k))
                break
            allocs.append(placed[0])
        else:
            crs[:] = shadow
            out.append(("placed", allocs))
    return out


def cr_occupancy(crs: list) -> np.ndarray:
    """The occupancy byte of every GPU in canonical order, rebuilt from the custom resources (:306-328)."""
    occ = []
    for cr in crs:
        for uuid in sorted(cr["spec"]["MigGPUUUID"]):
            b = 0
            for p in cr["spec"].get("prepared", {}).values():
                if p["parent"] == uuid and p["podUUID"] == "":
                    b |= ((1 << p["size"]) - 1) << p["start"]
            for a in cr["spec"].get("allocations", {}).values():
                if a["gpuUUID"] == uuid:
                    b |= ((1 << a["size"]) - 1) << a["start"]
            occ.append(b)
    return np.asarray(occ, dtype=np.uint8)
