"""CPU restatements of isl_place_gangs on an engine created with ISL_FLAG_GANG_LOCALITY (TEST INFRASTRUCTURE, NOT PRODUCT CODE): each
gang is placed by the locality its ALLOC members name in their ``start`` byte (include/islplace.h, L1-L6).  Two compositions that share
nothing but L2 (FREEs first, then the gangs in array order, each by the rules of its locality on the occupancy the earlier ones left):

``fast_gangs_locality``     every policy: the call's FREEs on a ``RangeFast``, then each run of consecutive gangs of one locality goes to
                            that locality's brute force, ``gang_oracle.fast_place_gangs`` on a ``RangeFast`` (0), ``gang_node_fast`` (1),
                            ``gang_few_fast`` (2) or ``gang_spread_fast`` (3), with the occupancy carried from one run to the next.
                            Returns the records and the occupancy after the call.
``ref_py_gangs_locality``   first-fit on CR-shaped dicts: each gang goes to the ``ref_py`` restatement of its locality,
                            ``gang_oracle.ref_py_place_gangs`` (0), ``gang_node_oracle`` (1), ``gang_few_oracle`` (2) or
                            ``gang_spread_oracle`` (3), on the same list of custom resources.
``load_kat``                the hand-worked vectors of tests/golden/kat_gang_locality.json as engine inputs.
"""
from __future__ import annotations

import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import gang_few_fast as GFF
import gang_few_oracle as GFO
import gang_node_fast as GNF
import gang_node_oracle as GNO
import gang_spread_fast as GSF
import gang_spread_oracle as GSO
from gang_oracle import default_sizes, fast_place_gangs, ref_py_place_gangs
from range_oracle import RangeFast

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_locality.json")
LOCALITIES = (E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_FEW_NODES, E.GANG_DISTINCT_NODES)
FLAG_OF = {E.GANG_ANY_NODES: 0, E.GANG_ONE_NODE: E.FLAG_GANG_ONE_NODE, E.GANG_FEW_NODES: E.FLAG_GANG_FEW_NODES,
           E.GANG_DISTINCT_NODES: E.FLAG_GANG_DISTINCT_NODES}
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "ABORTED": E.ST_GANG_ABORTED,
          "FREED": E.ST_FREED, "NOOP": E.ST_NOOP}


def with_locality(requests, gang_off, locality) -> np.ndarray:
    """A copy of ``requests`` whose ALLOC members carry their gang's locality in ``start`` (what ``Engine.place_gangs`` writes)."""
    req = np.array(requests, dtype=E.REQUEST_DTYPE)
    per = np.repeat(np.asarray(locality, dtype=np.int64), np.diff(np.asarray(gang_off, dtype=np.int64)))
    alloc = req["op"] == E.OP_ALLOC
    req["start"][alloc] = per[alloc].astype(np.uint8)
    return req


def gang_localities(requests, gang_off) -> list:
    """The locality of every gang (None for a gang without an ALLOC member)."""
    out = []
    for a, b in zip(gang_off[:-1], gang_off[1:]):
        idx = np.flatnonzero(requests["op"][a:b] == E.OP_ALLOC)
        out.append(int(requests["start"][a + idx[0]]) if len(idx) else None)
    return out


def fast_gangs_locality(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
                        lo=0, hi=None):
    node_off = np.asarray(node_off, dtype=np.uint32)
    rows = np.asarray(rows)
    hi = int(node_off[-1]) if hi is None else hi
    table = np.zeros(len(node_off) - 1, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    per_node = table if rows.ndim == 2 else None
    sizes = default_sizes(rows, table)
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.asarray(gang_off, dtype=np.int64)
    alloc = req["op"] == E.OP_ALLOC
    rest = req.copy()
    rest["op"][alloc] = E.OP_NOOP
    whole = RangeFast(node_off, rows, occ, lo, hi, quirks, policy, node_table=per_node)
    out = whole.place(rest)                         # every FREE first, NOOP records for the rest
    cur = whole.occupancy()
    runs = []                                       # [locality, [ALLOC member indices of each gang]]
    for a, b, loc in zip(gang_off[:-1], gang_off[1:], gang_localities(req, gang_off)):
        if loc is None:
            continue
        if not runs or runs[-1][0] != loc:
            runs.append([loc, []])
        runs[-1][1].append(np.flatnonzero(alloc[a:b]) + a)
    for loc, gangs in runs:
        idx = np.concatenate(gangs)
        members = req[idx].copy()
        members["start"] = 0
        off = np.cumsum([0] + [len(g) for g in gangs]).astype(np.uint32)
        if loc == E.GANG_ANY_NODES:
            run = RangeFast(node_off, rows, cur, lo, hi, quirks, policy, node_table=per_node)
            got = fast_place_gangs(run, members, off, sizes)
            cur = run.occupancy()
        else:
            brute = {E.GANG_ONE_NODE: GNF, E.GANG_FEW_NODES: GFF, E.GANG_DISTINCT_NODES: GSF}[loc]
            got, cur = brute.place_gangs(node_off, rows, cur, members, off, quirks, policy, node_table, lo, hi)
        out[idx] = got
    return out, np.asarray(cur, dtype=np.uint8)


def ref_py_gangs_locality(crs: list, gangs: list, locality: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``, ``locality`` one value per gang; ``crs`` one Instaslice dict per node, updated in
    place.  Returns per gang ("placed", [AllocationDetails...]) or ("aborted", index of the member that keeps its record)."""
    place = {E.GANG_ANY_NODES: ref_py_place_gangs, E.GANG_ONE_NODE: GNO.ref_py_gangs_one_node,
             E.GANG_FEW_NODES: GFO.ref_py_gangs_few_nodes, E.GANG_DISTINCT_NODES: GSO.ref_py_gangs_distinct_nodes}
    return [place[loc](crs, [gang], quirks)[0] for gang, loc in zip(gangs, locality)]


def kat_requests(gangs, names):
    """Requests and gang offsets of one vector: a member is a profile name or ["FREE", gpu, start, size]."""
    req = np.zeros(sum(len(g) for g in gangs), dtype=E.REQUEST_DTYPE)
    i = 0
    for g in gangs:
        for m in g:
            if isinstance(m, list):
                req[i] = (m[1], 0, E.OP_FREE, m[2], m[3])
            else:
                req[i] = (i, names.index(m) if m in names else E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
            i += 1
    return req, np.cumsum([0] + [len(g) for g in gangs]).astype(np.uint32)


def load_kat():
    """Yield per vector: (name, engine inputs dict, requests with their localities, gang offsets, expected records, expected occupancy)."""
    with open(KAT_PATH) as f:
        doc = json.load(f)
    for v in doc["vectors"]:
        tabs = [getattr(tables, t) for t in v["tables"]]
        if len(tabs) == 1:
            rows, names = E.make_profiles(tabs[0]), [r[0] for r in tabs[0]]
        else:
            names, rows = E.make_profile_tables(tabs)
            names = list(names)
        req, off = kat_requests(v["gangs"], names)
        req = with_locality(req, off, v["locality"])
        want = [(E.GPU_NONE if r[0] is None else r[0], r[1], r[2], STATUS[r[3]]) for g in v["records"] for r in g]
        inputs = {"node_off": np.asarray(v["node_off"], dtype=np.uint32), "rows": rows, "occ": np.asarray(v["occ"], dtype=np.uint8),
                  "policy": GFO.POLICY[v["policy"]], "quirks": E.QUIRKS_REF_EXACT if v["quirks"] == "ref_exact" else E.QUIRKS_FIXED,
                  "node_table": None if v.get("node_table") is None else np.asarray(v["node_table"], dtype=np.uint8),
                  "partition": v.get("partition"), "table_names": v["tables"], "names": names, "gangs": v["gangs"],
                  "locality": v["locality"]}
        yield v["name"], inputs, req, off, want, np.asarray(v["occ_after"], dtype=np.uint8)
