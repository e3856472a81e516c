"""CPU restatements of few-node gangs (isl_place_gangs with ISL_FLAG_GANG_FEW_NODES; TEST INFRASTRUCTURE, NOT PRODUCT CODE) that
share nothing with tests/gang_few_fast.cpp beyond the rules of include/islplace.h (F1-F6):

``ref_py_gangs_few_nodes``  first-fit on CR-shaped dicts: per round, ``ref_py.reconcile_gated_pod`` member by member from the first
                            unplaced member on a deep copy of each node's custom resource, node after node in list order; the copy that
                            placed the most (the first on a tie) replaces the node's resource.  A round that places nothing puts back
                            every resource the gang touched.  Returns per gang ("placed", [AllocationDetails...]) or ("aborted", i).
``fast_gangs_few_nodes``    every policy: per round and per node of the range in scan order, a ``RangeFast`` over that node's GPUs
                            composed with ``gang_oracle.fast_place_gangs`` on the remaining members; the depth of each node is where its
                            gang came back aborted.  Returns the records and the occupancy after the call.
``load_kat``                the hand-worked vectors of tests/golden/kat_gang_few.json as engine inputs.
"""
from __future__ import annotations

import copy
import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables
from oracle import ref_py

from gang_oracle import default_sizes, fast_place_gangs
from range_oracle import RangeFast

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_few.json")
POLICY = {"first_fit": E.POLICY_FIRST_FIT, "best_fit": E.POLICY_BEST_FIT, "right_to_left": E.POLICY_RIGHT_TO_LEFT,
          "min_frag": E.POLICY_MIN_FRAG}
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "ABORTED": E.ST_GANG_ABORTED}


def ref_py_gangs_few_nodes(crs: list, gangs: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``; ``crs`` one Instaslice dict per node, updated in place."""
    out = []
    for gang in gangs:
        before = copy.deepcopy(crs)
        allocs = []
        while len(allocs) < len(gang):
            best, best_n, best_allocs = None, -1, []
            for n in range(len(crs)):
                shadow = [copy.deepcopy(crs[n])]
                placed = []
                for pod, name in gang[len(allocs):]:
                    verdict, got = ref_py.reconcile_gated_pod(shadow, pod, name, quirks)
                    if verdict != "placed":
                        break
                    placed.append(got[0])
                if len(placed) > len(best_allocs):
                    best, best_n, best_allocs = shadow[0], n, placed
            if not best_allocs:
                break
            crs[best_n] = best
            allocs += best_allocs
        if len(allocs) == len(gang):
            out.append(("placed", allocs))
        else:
            crs[:] = before
            out.append(("aborted", len(allocs)))
    return out


def fast_gangs_few_nodes(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT,
                         node_table=None, lo=0, hi=None):
    node_off = np.asarray(node_off, dtype=np.int64)
    rows = np.asarray(rows)
    n_nodes = len(node_off) - 1
    hi = int(node_off[-1]) if hi is None else hi
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    per_node = table if rows.ndim == 2 else None
    sizes = default_sizes(rows, table)
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    alloc = req["op"] == E.OP_ALLOC
    whole = RangeFast(node_off, rows, occ, lo, hi, quirks, policy, node_table=per_node)
    rest = req.copy()
    rest["op"][alloc] = E.OP_NOOP
    out = whole.place(rest)                         # every FREE first, NOOP records for the rest
    for i in np.flatnonzero(alloc):                 # default records of the ALLOCs
        p = int(req["profile"][i])
        out[i] = (E.GPU_NONE, E.START_NONE, sizes[p], E.ST_NO_CAPACITY) if p < len(sizes) else (E.GPU_NONE, E.START_NONE, 0, E.ST_BAD_PROFILE)
    cur = whole.occupancy()
    order = range(n_nodes - 1, -1, -1) if policy == E.POLICY_RIGHT_TO_LEFT else range(n_nodes)
    for a, b in zip(gang_off[:-1], gang_off[1:]):
        idx = np.flatnonzero(alloc[a:b]) + a
        if len(idx) == 0:
            continue
        work, got, m = cur, np.zeros(len(idx), dtype=E.RESULT_DTYPE), 0
        while m < len(idx):
            best_d, best_node = 0, None
            for n in order:
                nlo, nhi = max(int(node_off[n]), lo), min(int(node_off[n + 1]), hi)
                if nlo >= nhi:
                    continue
                one = RangeFast(node_off, rows, work, nlo, nhi, quirks, policy, node_table=per_node)
                res = fast_place_gangs(one, req[idx[m:]], [0, len(idx) - m], sizes)
                bad = np.flatnonzero(res["status"] != E.ST_PLACED)
                d = len(res) if len(bad) == 0 else int(np.flatnonzero(res["status"] != E.ST_GANG_ABORTED)[0])
                if d > best_d:
                    best_d, best_node = d, (nlo, nhi)
            if best_d == 0:
                break
            one = RangeFast(node_off, rows, work, best_node[0], best_node[1], quirks, policy, node_table=per_node)
            got[m:m + best_d] = fast_place_gangs(one, req[idx[m:m + best_d]], [0, best_d], sizes)
            work = one.occupancy()
            m += best_d
        if m == len(idx):
            out[idx] = got
            cur = work
            continue
        for k, i in enumerate(idx):
            if k != m:
                p = int(req["profile"][i])
                out[i] = (E.GPU_NONE, E.START_NONE, sizes[p] if p < len(sizes) else 0, E.ST_GANG_ABORTED)
    return out, cur


def load_kat():
    """Yield per vector: (name, engine inputs dict, gangs of profile indices, expected records per gang, expected occupancy)."""
    with open(KAT_PATH) as f:
        doc = json.load(f)
    for v in doc["vectors"]:
        tabs = [getattr(tables, t) for t in v["tables"]]
        if len(tabs) == 1:
            rows, names = E.make_profiles(tabs[0]), [r[0] for r in tabs[0]]
        else:
            names, rows = E.make_profile_tables(tabs)
            names = list(names)
        index = lambda name: names.index(name) if name in names else E.PROFILE_UNKNOWN  # noqa: E731
        gangs = [[index(x) for x in g] for g in v["gangs"]]
        want = [[(E.GPU_NONE if r[0] is None else r[0], r[1], r[2], STATUS[r[3]]) for r in g] for g in v["records"]]
        inputs = {"node_off": np.asarray(v["node_off"], dtype=np.uint32), "rows": rows, "occ": np.asarray(v["occ"], dtype=np.uint8),
                  "policy": POLICY[v["policy"]], "quirks": E.QUIRKS_REF_EXACT if v["quirks"] == "ref_exact" else E.QUIRKS_FIXED,
                  "node_table": None if v.get("node_table") is None else np.asarray(v["node_table"], dtype=np.uint8),
                  "partition": v.get("partition"), "table_names": v["tables"]}
        yield v["name"], inputs, gangs, want, np.asarray(v["occ_after"], dtype=np.uint8)
