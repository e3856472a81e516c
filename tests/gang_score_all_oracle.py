"""Every gang kind under node scoring (isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_NODE_SCORE_ALL engine,
include/islplace.h C1-C8) restated on top of the unchanged single-pod checker ``node_score_fast.place`` (ns) and the node-scored gang
checker ``gang_score_oracle.place_gangs``, sharing nothing with tests/gang_score_all_fast.cpp but the rules:

- any node and distinct nodes (bytes 0 and 3): ``gang_score_oracle.place_gangs`` on the gang alone (N3, N4);
- balanced (bytes 4..255): per member, one ns call per node with the node alone as the range tells which nodes admit it; mu is their
  least count, and one ns call over the whole range on a copy in which the nodes above mu + k - 1 are full (0xFF) places it (C6);
- one node and few nodes (bytes 1 and 2): per round one ns call per node with the node alone as the range (node scoring is first-fit
  there); its leading PLACED records are d, their sizes R_d; the deepest node wins, then the best score for R_d, then the lowest node
  (N5, C4);
- elastic: a gang that stops at ALLOC member f >= m' is run again cut to its first f members, which must commit (M5 b, C5).

Also the known-answer vectors of tests/golden/kat_gang_score_all.json.
"""
from __future__ import annotations

import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import gang_score_oracle as GSO
import node_score_fast as NS
from gang_locality_oracle import gang_localities
from gang_min_fast import effective_minimum

KAT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_score_all.json")
STATUS = dict(GSO.STATUS, GANG_TRIMMED=E.ST_GANG_TRIMMED)
PER_GANG = None


def _busy(occ, a, b, w):
    return sum(bin(int(x) & ((1 << w) - 1)).count("1") for x in occ[a:b])


def _ones(got):
    """How many leading records are PLACED."""
    return next((k for k, g in enumerate(got) if g["status"] != E.ST_PLACED), len(got))


def _apply(occ, recs):
    for r in recs:
        occ[int(r["gpu"])] |= ((1 << int(r["size"])) - 1) << int(r["start"])


def place_gangs(node_off, rows, occ, requests, gang_off, policy, locality=PER_GANG, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0,
                hi=None, elastic=False):
    """(records, occupancy after, members placed) as gang_score_all_fast.place_gangs returns them."""
    node_off = np.asarray(node_off, dtype=np.uint32)
    rows2 = np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1])
    n_nodes = len(node_off) - 1
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    width = GSO.widths(rows2)
    hi = int(node_off[-1]) if hi is None else hi
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.asarray(gang_off, dtype=np.int64)
    out = np.zeros(len(req), dtype=E.RESULT_DTYPE)
    spans = [(v, max(int(node_off[v]), lo), min(int(node_off[v + 1]), hi)) for v in range(n_nodes)]
    spans = [s for s in spans if s[1] < s[2]]

    def ns(o, sub, a=lo, b=hi):
        return NS.place(node_off, rows2, o, sub, policy, quirks=quirks, node_table=table, lo=a, hi=b)

    other = req["op"] != E.OP_ALLOC                                 # rule 1: FREEs first, NOOPs report NOOP
    out[other], cur = ns(occ, req[other])
    allocs = np.flatnonzero(~other)
    out[allocs] = ns(cur, req[allocs], 0, 0)[0]                     # the default records: an empty range places nothing
    locs = gang_localities(req, gang_off) if locality is PER_GANG else [locality] * (len(gang_off) - 1)
    mins = effective_minimum(req, gang_off) if elastic else None

    def run(members, loc, o):
        """The ALLOC ``members`` of one gang by its locality on occupancy ``o``: (records of the leading members it placed, occupancy
        with them)."""
        o = np.array(o, dtype=np.uint8)
        if loc in (E.GANG_ANY_NODES, E.GANG_DISTINCT_NODES):
            got, after, _ = GSO.place_gangs(node_off, rows2, o, members, [0, len(members)], policy, loc, quirks, table, lo, hi)
            if (got["status"] == E.ST_PLACED).all():
                return list(got), after
            return [None] * int(np.flatnonzero(got["status"] != E.ST_GANG_ABORTED)[0]), o     # rule 4: only f counts
        if loc > E.GANG_DISTINCT_NODES:
            skew, cnt, recs = loc - E.GANG_DISTINCT_NODES, [0] * n_nodes, []
            for i in range(len(members)):
                admit = [v for v, a, b in spans if ns(o, members[i:i + 1], a, b)[0][0]["status"] == E.ST_PLACED]
                if not admit:
                    break
                mu = min(cnt[v] for v in admit)
                view = o.copy()
                for v, a, b in spans:
                    if cnt[v] > mu + skew - 1:
                        view[a:b] = 0xFF
                got = ns(view, members[i:i + 1])[0][0]
                recs.append(got)
                _apply(o, [got])
                cnt[next(v for v, a, b in spans if a <= int(got["gpu"]) < b)] += 1
            return recs, o
        recs = []
        while len(recs) < len(members):
            best = None                                             # (d, score, -node, records)
            for v, a, b in spans:
                got = ns(o, members[len(recs):], a, b)[0]
                d = _ones(got)
                if d == 0:
                    continue
                w = width[table[v]]
                s = GSO.score(policy, w * (b - a), _busy(o, a, b, w), int(got["size"][:d].sum()))
                if best is None or (d, s, -v) > best[:3]:
                    best = (d, s, -v, list(got[:d]))
            if best is None:
                break
            recs += best[3]
            _apply(o, best[3])
            if loc == E.GANG_ONE_NODE:
                break
        return recs, o

    placed = 0
    for g, (a, b) in enumerate(zip(gang_off[:-1], gang_off[1:])):
        idx = np.flatnonzero(req["op"][a:b] == E.OP_ALLOC) + a
        if not len(idx):
            continue
        recs, after = run(req[idx], locs[g], cur)
        f, k = len(recs), len(idx)
        if f == k:
            out[idx], cur = recs, after
            placed += k
            continue
        if elastic and f >= int(mins[g]):                           # M5 (b): the gang cut to its first f members commits
            cut, cur = run(req[idx[:f]], locs[g], cur)
            assert len(cut) == f, "a gang cut at the member it failed at must commit"
            out[idx[:f]] = cut
            out["status"][idx[f + 1:]] = E.ST_GANG_TRIMMED
            placed += f
        else:                                                       # member f keeps its default record
            out["status"][np.delete(idx, f)] = E.ST_GANG_ABORTED
    return out, np.asarray(cur, dtype=np.uint8), placed


# ---- known-answer vectors --------------------------------------------------------------------------------------------------------------
def kat_vectors():
    with open(KAT) as f:
        return json.load(f)["vectors"]


def vector_inputs(v):
    """The engine inputs of one vector: a dict of node_off, rows, node_table, occ, requests, gang_off, quirks, policy, lo, hi, the engine
    locality (None: each gang's byte, FLAG_GANG_LOCALITY) and elastic.  A table is a name of instaslice_b200.tables; a request is
    [profile name or "NOOP" or ["FREE", gpu, start, size], start byte, size byte]; gangs: the number of requests of every gang."""
    names, rows = E.make_profile_tables([tables.TABLES[t] for t in v["tables"]])
    req = np.zeros(len(v["requests"]), dtype=E.REQUEST_DTYPE)
    for i, (p, b, m) in enumerate(v["requests"]):
        if isinstance(p, list):
            req[i]["handle"], req[i]["op"], req[i]["start"], req[i]["size"] = p[1], E.OP_FREE, p[2], p[3]
            continue
        req[i]["op"] = E.OP_NOOP if p == "NOOP" else E.OP_ALLOC
        req[i]["profile"] = 0 if p == "NOOP" else names.index(p) if p in names else E.PROFILE_UNKNOWN
        req[i]["start"], req[i]["size"] = b, m
    node_off = np.array(v["node_off"], dtype=np.uint32)
    return {"node_off": node_off, "rows": rows, "node_table": np.array(v["node_table"], dtype=np.uint8),
            "occ": np.array(v["occ"], dtype=np.uint8), "requests": req, "gang_off": np.cumsum([0] + v["gangs"]).astype(np.uint32),
            "quirks": GSO.QUIRKS[v["quirks"]], "policy": GSO.POLICY[v["policy"]], "lo": v.get("lo", 0),
            "hi": v.get("hi", int(node_off[-1])), "locality": v["locality"], "elastic": v["elastic"]}


def expected(v):
    recs = [(E.GPU_NONE if g is None else g, s, z, STATUS[st]) for g, s, z, st in v["records"]]
    return recs, np.array(v["occ_after"], dtype=np.uint8), v["placed"]


def run_vector(checker, x):
    return checker(x["node_off"], x["rows"], x["occ"], x["requests"], x["gang_off"], x["policy"], x["locality"], quirks=x["quirks"],
                   node_table=x["node_table"], lo=x["lo"], hi=x["hi"], elastic=x["elastic"])
