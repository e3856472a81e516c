"""CPU restatements of one-node gangs (isl_place_gangs with ISL_FLAG_GANG_ONE_NODE; TEST INFRASTRUCTURE, NOT PRODUCT CODE) that
share nothing with tests/gang_node_fast.cpp beyond the rules of include/islplace.h:

``ref_py_gangs_one_node``  first-fit on CR-shaped dicts: ``ref_py.reconcile_gated_pod`` member by member on a deep copy of ONE node's
                           custom resource, node after node in list order; the first copy that places every member replaces the node's
                           resource.  Returns per gang ("placed", [AllocationDetails...]) or ("aborted", D).
``fast_gangs_one_node``    every policy: per node of the range in scan order, a ``RangeFast`` over that node's GPUs composed with
                           ``gang_oracle.fast_place_gangs``; the first node whose gang comes back placed is kept.  Returns the records
                           and the occupancy after the call.
``load_kat``               the hand-worked vectors of tests/golden/kat_gang_node.json as engine inputs.
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

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_node.json")
POLICY = {"first_fit": E.POLICY_FIRST_FIT, "best_fit": E.POLICY_BEST_FIT, "right_to_left": E.POLICY_RIGHT_TO_LEFT,
          "min_frag": E.POLICY_MIN_FRAG}
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "ABORTED": E.ST_GANG_ABORTED}


def ref_py_gangs_one_node(crs: list, gangs: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``; ``crs`` one Instaslice dict per node, updated in place."""
    out = []
    for gang in gangs:
        deepest, done = 0, False
        for n in range(len(crs)):
            shadow = [copy.deepcopy(crs[n])]
            allocs = []
            for pod, name in gang:
                verdict, placed = ref_py.reconcile_gated_pod(shadow, pod, name, quirks)
                if verdict != "placed":
                    break
                allocs.append(placed[0])
            if len(allocs) == len(gang):
                crs[n] = shadow[0]
                out.append(("placed", allocs))
                done = True
                break
            deepest = max(deepest, len(allocs))
        if not done:
            out.append(("aborted", deepest))
    return out


def fast_gangs_one_node(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT,
                        node_table=None, lo=0, hi=None):
    node_off = np.asarray(node_off, dtype=np.int64)
    rows = np.asarray(rows)
    n_nodes = len(node_off) - 1
    hi = int(node_off[-1]) if hi is None else hi
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    sizes = default_sizes(rows, table)
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    alloc = req["op"] == E.OP_ALLOC
    whole = RangeFast(node_off, rows, occ, lo, hi, quirks, policy, node_table=table if rows.ndim == 2 else None)
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
        deepest, done = 0, False
        for n in order:
            nlo, nhi = max(int(node_off[n]), lo), min(int(node_off[n + 1]), hi)
            if nlo >= nhi:
                continue
            one = RangeFast(node_off, rows, cur, nlo, nhi, quirks, policy, node_table=table if rows.ndim == 2 else None)
            res = fast_place_gangs(one, req[idx], [0, len(idx)], sizes)
            failed = np.flatnonzero(res["status"] != E.ST_PLACED)
            if len(failed) == 0:
                out[idx] = res
                cur = one.occupancy()
                done = True
                break
            deepest = max(deepest, int(np.flatnonzero(res["status"] != E.ST_GANG_ABORTED)[0]))     # the member that found nothing
        if done:
            continue
        for k, i in enumerate(idx):
            if k != deepest:
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
