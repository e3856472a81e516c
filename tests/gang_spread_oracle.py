"""CPU restatements of distinct-node gangs (isl_place_gangs with ISL_FLAG_GANG_DISTINCT_NODES; TEST INFRASTRUCTURE, NOT PRODUCT CODE)
that share nothing with tests/gang_spread_fast.cpp beyond the rules of include/islplace.h:

``ref_py_gangs_distinct_nodes``  first-fit on CR-shaped dicts: ``ref_py.reconcile_gated_pod`` member by member on a deep copy of the
                                 cluster that hides the nodes the gang already uses; a gang whose members all come back "placed"
                                 replaces the cluster with the copy.  Returns per gang ("placed", [AllocationDetails...]) or
                                 ("aborted", index of the member that found nothing).
``fast_gangs_distinct_nodes``    every policy: per member, each unused node of the range proposes its own choice (a ``RangeFast`` over
                                 that node's GPUs), and the proposals are compared by (policy score, scan position).  Returns the
                                 records and the occupancy after the call.
``load_kat``                     the hand-worked vectors of tests/golden/kat_gang_spread.json as engine inputs.
"""
from __future__ import annotations

import copy
import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables
from oracle import ref_py

from gang_oracle import default_sizes
from range_oracle import RangeFast

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_spread.json")
POLICY = {"first_fit": E.POLICY_FIRST_FIT, "best_fit": E.POLICY_BEST_FIT, "right_to_left": E.POLICY_RIGHT_TO_LEFT,
          "min_frag": E.POLICY_MIN_FRAG}
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "ABORTED": E.ST_GANG_ABORTED,
          "FREED": E.ST_FREED, "NOOP": E.ST_NOOP}


def ref_py_gangs_distinct_nodes(crs: list, gangs: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``; ``crs`` one Instaslice dict per node, updated in place."""
    out = []
    for gang in gangs:
        shadow = copy.deepcopy(crs)
        used, allocs = set(), []
        for k, (pod, name) in enumerate(gang):
            visible = [cr for n, cr in enumerate(shadow) if n not in used]
            verdict, placed = ref_py.reconcile_gated_pod(visible, pod, name, quirks)
            if verdict != "placed":
                out.append(("aborted", k))
                break
            used.add(next(n for n, cr in enumerate(shadow) if placed[0]["gpuUUID"] in cr["spec"]["MigGPUUUID"]))
            allocs.append(placed[0])
        else:
            crs[:] = shadow
            out.append(("placed", allocs))
    return out


def _legal(size, v, quirks):
    """Slot mask of ``size`` slices at start ``v`` under the quirk set, 0 when the start search never returns it (:343-383)."""
    size, v = int(size), int(v)
    if v >= 8 or size == 0 or size > 8:
        return 0
    if size == 1:
        return 1 << v
    if quirks & E.QUIRK_POW2_ONLY and size not in (2, 4, 8):
        return 0
    if (v + size >= 8) if quirks & E.QUIRK_STRICT_BOUND else (v + size > 8):
        return 0
    return ((1 << size) - 1) << v


def _score(policy, table_rows, quirks, o, mine):
    """What the policy minimises when ``mine`` is taken on byte ``o`` of a GPU whose node uses ``table_rows``."""
    if policy == E.POLICY_BEST_FIT:
        return 8 - bin(o | mine).count("1")
    if policy != E.POLICY_MIN_FRAG:
        return 0
    masks = [_legal(r["size"], s, quirks) for r in table_rows for s in r["starts"][:r["n_starts"]]]
    return sum(1 for m in masks if m and o & m == 0 and (o | mine) & m)


def fast_gangs_distinct_nodes(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT,
                              node_table=None, lo=0, hi=None):
    node_off = np.asarray(node_off, dtype=np.int64)
    rows = np.asarray(rows)
    n_nodes, G = len(node_off) - 1, int(node_off[-1])
    hi = G if hi is None else hi
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    per_node = table if rows.ndim == 2 else None
    sizes = default_sizes(rows, table)
    n_profiles = rows.shape[-1]
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    alloc = req["op"] == E.OP_ALLOC
    whole = RangeFast(node_off, rows, occ, lo, hi, quirks, policy, node_table=per_node)
    rest = req.copy()
    rest["op"][alloc] = E.OP_NOOP
    out = whole.place(rest)                         # every FREE first, NOOP records for the rest
    for i in np.flatnonzero(alloc):                 # default records of the ALLOCs
        p = int(req["profile"][i])
        out[i] = (E.GPU_NONE, E.START_NONE, sizes[p], E.ST_NO_CAPACITY) if p < n_profiles else (E.GPU_NONE, E.START_NONE, 0, E.ST_BAD_PROFILE)
    cur = whole.occupancy()
    descending = policy == E.POLICY_RIGHT_TO_LEFT
    for a, b in zip(gang_off[:-1], gang_off[1:]):
        idx = np.flatnonzero(alloc[a:b]) + a
        tent, used, got = cur.copy(), set(), []
        for i in idx:
            best = None                             # ((score, scan position), record, node)
            if int(req["profile"][i]) < n_profiles:
                for n in range(n_nodes):
                    nlo, nhi = max(int(node_off[n]), lo), min(int(node_off[n + 1]), hi)
                    if n in used or nlo >= nhi:
                        continue
                    r = RangeFast(node_off, rows, tent, nlo, nhi, quirks, policy, node_table=per_node).place(req[i:i + 1])[0]
                    if r["status"] != E.ST_PLACED:
                        continue
                    g, mine = int(r["gpu"]), ((1 << int(r["size"])) - 1) << int(r["start"])
                    key = (_score(policy, rows[table[n]] if rows.ndim == 2 else rows, quirks, int(tent[g]), mine),
                           G - 1 - g if descending else g)
                    if best is None or key < best[0]:
                        best = (key, r, n)
            if best is None:
                break
            _key, r, n = best
            tent[int(r["gpu"])] |= ((1 << int(r["size"])) - 1) << int(r["start"])
            used.add(n)
            got.append(r)
        if len(got) == len(idx):
            for i, r in zip(idx, got):
                out[i] = r
            cur = tent
            continue
        for k, i in enumerate(idx):                 # the member at len(got) found nothing and keeps its record
            if k != len(got):
                p = int(req["profile"][i])
                out[i] = (E.GPU_NONE, E.START_NONE, sizes[p] if p < n_profiles else 0, E.ST_GANG_ABORTED)
    return out, cur


def load_kat():
    """Yield per vector: (name, engine inputs dict, per gang its requests, expected records per gang, expected occupancy, profile names
    per gang or None when a gang holds a FREE or a NOOP).  A member is a profile name, "NOOP", or {"free": [gpu, start, size]}."""
    with open(KAT_PATH) as f:
        doc = json.load(f)
    for v in doc["vectors"]:
        tabs = [getattr(tables, t) for t in v["tables"]]
        if len(tabs) == 1:
            rows, names = E.make_profiles(tabs[0]), [r[0] for r in tabs[0]]
        else:
            names, rows = E.make_profile_tables(tabs)
            names = list(names)
        gangs, plain = [], []
        for g in v["gangs"]:
            req = np.zeros(len(g), dtype=E.REQUEST_DTYPE)
            for k, m in enumerate(g):
                if isinstance(m, dict):
                    req[k] = (m["free"][0], 0, E.OP_FREE, m["free"][1], m["free"][2])
                elif m == "NOOP":
                    req[k] = (0, 0, E.OP_NOOP, 0, 0)
                else:
                    req[k] = (k, names.index(m) if m in names else E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
            gangs.append(req)
            plain.append(g if all(isinstance(m, str) and m != "NOOP" for m in g) else None)
        want = [[(E.GPU_NONE if r[0] is None else r[0], r[1], r[2], STATUS[r[3]]) for r in g] for g in v["records"]]
        inputs = {"node_off": np.asarray(v["node_off"], dtype=np.uint32), "rows": rows, "occ": np.asarray(v["occ"], dtype=np.uint8),
                  "policy": POLICY[v["policy"]], "quirks": E.QUIRKS_REF_EXACT if v["quirks"] == "ref_exact" else E.QUIRKS_FIXED,
                  "node_table": None if v.get("node_table") is None else np.asarray(v["node_table"], dtype=np.uint8),
                  "partition": v.get("partition"), "table_names": v["tables"], "profile_names": names}
        yield v["name"], inputs, gangs, want, np.asarray(v["occ_after"], dtype=np.uint8), plain
