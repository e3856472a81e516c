"""Node-scored gangs (isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE engine, include/islplace.h N1-N8) restated on top of the unchanged
single-pod checker ``node_score_fast.place`` (ns_place), sharing nothing with tests/gang_score_fast.cpp but the rules:

- any node: the ALLOC members one ns_place call each on a copy of the occupancy, kept when every member is PLACED, dropped otherwise;
- distinct nodes: the same, each member placed on a copy in which the nodes of the gang's earlier members are full (0xFF);
- one node: one ns_place call per node with the node alone as the range (node scoring is first-fit there), then the gang's score from
  the rules, the slices its members take counted as one pod.

Also the known-answer cases of tests/golden/kat_gang_score.json and the random clusters the CPU and GPU tests share.
"""
from __future__ import annotations

import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import node_score_fast as NS

KAT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_score.json")
QUIRKS = {"REF_EXACT": E.QUIRKS_REF_EXACT, "FIXED": E.QUIRKS_FIXED}
POLICY = {"MOST_ALLOCATED": E.POLICY_MOST_ALLOCATED, "LEAST_ALLOCATED": E.POLICY_LEAST_ALLOCATED}
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "NOOP": E.ST_NOOP,
          "FREED": E.ST_FREED, "GANG_ABORTED": E.ST_GANG_ABORTED}
PER_GANG = 4
LOCALITY = {"ANY": E.GANG_ANY_NODES, "ONE": E.GANG_ONE_NODE, "DISTINCT": E.GANG_DISTINCT_NODES, "PER_GANG": PER_GANG}
FLAGS = {E.GANG_ANY_NODES: 0, E.GANG_ONE_NODE: E.FLAG_GANG_ONE_NODE, E.GANG_DISTINCT_NODES: E.FLAG_GANG_DISTINCT_NODES,
         PER_GANG: E.FLAG_GANG_LOCALITY}


def widths(rows2):
    """Node-scoring rule 2: the width of every table, the largest start + size of its rows."""
    return [max([int(r["starts"][k]) + int(r["size"]) for r in rows2[t] for k in range(int(r["n_starts"]))] or [0])
            for t in range(rows2.shape[0])]


def score(policy, cap, busy, req):
    return 100 * (busy + req) // cap if policy == E.POLICY_MOST_ALLOCATED else 100 * (cap - busy - req) // cap


def place_gangs(node_off, rows, occ, requests, gang_off, policy, locality, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0, hi=None):
    """(records, occupancy after, members placed) as gang_score_fast.place_gangs returns them, built from ns_place calls only."""
    node_off = np.asarray(node_off, dtype=np.uint32)
    rows2 = np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1])
    n_nodes = len(node_off) - 1
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    width = widths(rows2)
    hi = int(node_off[-1]) if hi is None else hi
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    out = np.zeros(len(req), dtype=E.RESULT_DTYPE)

    def ns(o, sub, a=lo, b=hi):
        return NS.place(node_off, rows2, o, sub, policy, quirks=quirks, node_table=table, lo=a, hi=b)

    other = req["op"] != E.OP_ALLOC                                 # rule 1: FREEs first, NOOPs report NOOP
    out[other], occ = ns(occ, req[other])
    allocs = np.flatnonzero(~other)
    unplaced = ns(occ, req[allocs], 0, 0)[0]                        # the default records: an empty range places nothing
    out[allocs] = unplaced
    default = dict(zip(allocs.tolist(), unplaced))
    placed = 0
    for r0, r1 in zip(gang_off[:-1], gang_off[1:]):
        members = [i for i in range(int(r0), int(r1)) if req[i]["op"] == E.OP_ALLOC]
        if not members:
            continue
        loc = int(req[members[0]]["start"]) if locality == PER_GANG else locality
        recs, fail = [], None
        if loc == E.GANG_ONE_NODE:
            best, deepest = None, 0
            for v in range(n_nodes):
                a, b = max(int(node_off[v]), lo), min(int(node_off[v + 1]), hi)
                if a >= b:
                    continue
                got, _ = ns(occ, req[members], a, b)
                d = next((k for k, g in enumerate(got) if g["status"] != E.ST_PLACED), len(members))
                deepest = max(deepest, d)
                if d < len(members):
                    continue
                w = width[table[v]]
                busy = sum(bin(int(x) & ((1 << w) - 1)).count("1") for x in occ[a:b])
                s = score(policy, w * (b - a), busy, int(got["size"].sum()))
                if best is None or s > best[0]:
                    best = (s, got)
            if best is None:
                fail = deepest
            else:
                recs = list(best[1])
        else:
            work = occ.copy()
            used = []
            for k, i in enumerate(members):
                view = work.copy()
                for v in used if loc == E.GANG_DISTINCT_NODES else []:
                    view[node_off[v]:node_off[v + 1]] = 0xFF
                got, after = ns(view, req[i:i + 1])
                if got[0]["status"] != E.ST_PLACED:
                    fail = k
                    break
                g = int(got[0]["gpu"])
                work[g] = after[g]
                used.append(int(np.searchsorted(node_off, g, side="right")) - 1)
                recs.append(got[0])
        if fail is None:
            for i, rec in zip(members, recs):
                out[i] = rec
                occ[rec["gpu"]] |= ((1 << int(rec["size"])) - 1) << int(rec["start"])
            placed += len(members)
            continue
        for k, i in enumerate(members):
            if k != fail:
                p = int(req[i]["profile"])
                out[i] = (E.GPU_NONE, 9, int(default[i]["size"]) if p < rows2.shape[1] else 0, E.ST_GANG_ABORTED)
    return out, occ, placed


# ---- known-answer cases ----------------------------------------------------------------------------------------------------------------
def kat_cases():
    with open(KAT) as f:
        return json.load(f)["cases"]


def case_inputs(case):
    """node_off, rows [n_tables][n_names], node_table, occ, requests, gang_off, quirks, policy, lo, hi, locality of a case.  A table is
    a name of instaslice_b200.tables or its rows [name, size, starts, gi]; a request is [profile name or "NOOP" or ["FREE", gpu, start,
    size], start byte]; gangs: the number of requests of every gang."""
    names, rows = E.make_profile_tables([tables.TABLES[t] if isinstance(t, str) else [tuple(r) for r in t] for t in case["tables"]])
    req = np.zeros(len(case["requests"]), dtype=E.REQUEST_DTYPE)
    for i, (p, b) in enumerate(case["requests"]):
        if isinstance(p, list):
            req[i]["handle"], req[i]["op"], req[i]["start"], req[i]["size"] = p[1], E.OP_FREE, p[2], p[3]
            continue
        req[i]["op"] = E.OP_NOOP if p == "NOOP" else E.OP_ALLOC
        req[i]["profile"] = 0 if p == "NOOP" else names.index(p) if p in names else E.PROFILE_UNKNOWN
        req[i]["start"] = b
    node_off = np.array(case["node_off"], dtype=np.uint32)
    gang_off = np.cumsum([0] + case["gangs"]).astype(np.uint32)
    return (node_off, rows, np.array(case["node_table"], dtype=np.uint8), np.array(case["occ"], dtype=np.uint8), req, gang_off,
            QUIRKS[case["quirks"]], POLICY[case["policy"]], case.get("lo", 0), case.get("hi", int(node_off[-1])), LOCALITY[case["locality"]])


def expected(case):
    recs = [(E.GPU_NONE if g is None else g, s, z, STATUS[st]) for g, s, z, st in case["records"]]
    return recs, np.array(case["occ_after"], dtype=np.uint8)


# ---- random clusters -------------------------------------------------------------------------------------------------------------------
def random_rows(rnd, n_tables=None):
    """[n_tables][n_names] rows of 1..3 reference tables."""
    while True:                                                  # an engine loads at most 16 profile names
        picked = rnd.sample(list(tables.TABLES), n_tables or rnd.randint(1, 3))
        names, rows = E.make_profile_tables([tables.TABLES[t] for t in picked])
        if len(names) <= E.MAX_PROFILES:
            return names, rows


def random_case(rnd, n_gpus, n_req, rows, max_gang=4, locality=None, policy=None, quirks=None, partition=True, max_nodes=12):
    """A random cluster and gang burst with FREEs, NOOPs and unknown profiles: (inputs as case_inputs returns them)."""
    n_tables, n_prof = rows.shape[0], rows.shape[1]
    n_nodes = rnd.randint(1, max(1, min(n_gpus, max_nodes)))
    cuts = sorted(rnd.sample(range(1, n_gpus), n_nodes - 1)) if n_nodes > 1 else []
    node_off = np.array([0] + cuts + [n_gpus], dtype=np.uint32)
    node_table = np.array([rnd.randrange(n_tables) for _ in range(n_nodes)], dtype=np.uint8)
    occ = np.array([rnd.choice([0, 0, 0x01, 0x03, 0x0F, 0x30, 0x81, 0xF0, rnd.randrange(256)]) for _ in range(n_gpus)], dtype=np.uint8)
    locality = rnd.choice([0, 1, 3, PER_GANG]) if locality is None else locality
    req = np.zeros(n_req, dtype=E.REQUEST_DTYPE)
    sizes = []
    while sum(sizes) < n_req:
        sizes.append(min(n_req - sum(sizes), rnd.randint(1, max_gang)))
    i = 0
    for k in sizes:
        lb = rnd.choice([0, 1, 3])
        for r in range(i, i + k):
            u = rnd.random()
            if u < 0.05:
                req[r]["op"], req[r]["handle"] = E.OP_FREE, rnd.randrange(n_gpus + 1)
                req[r]["start"], req[r]["size"] = rnd.randrange(8), rnd.randint(1, 4)
                continue
            req[r]["op"] = E.OP_NOOP if u < 0.09 else E.OP_ALLOC
            req[r]["profile"] = E.PROFILE_UNKNOWN if u > 0.98 else rnd.randrange(n_prof)
            req[r]["start"] = lb if locality == PER_GANG else rnd.randrange(9)
        i += k
    gang_off = np.cumsum([0] + sizes).astype(np.uint32)
    lo, hi = 0, n_gpus
    if partition and rnd.random() < 0.3 and n_gpus > 1:
        lo = rnd.randrange(n_gpus)
        hi = rnd.randint(lo + 1, n_gpus)
    policy = rnd.choice([E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]) if policy is None else policy
    quirks = rnd.choice([E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED]) if quirks is None else quirks
    return node_off, rows, node_table, occ, req, gang_off, quirks, policy, lo, hi, locality


def run(checker, inputs):
    node_off, rows, node_table, occ, req, gang_off, quirks, policy, lo, hi, loc = inputs
    return checker(node_off, rows, occ, req, gang_off, policy, loc, quirks=quirks, node_table=node_table, lo=lo, hi=hi)
