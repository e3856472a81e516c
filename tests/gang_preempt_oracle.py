"""Gang preemption (isl_preempt on an ISL_FLAG_GANG_PREEMPT engine, include/islplace.h P1-P8) restated on top of the unchanged
single-pod checker ``preempt_fast.preempt`` (pf_preempt), sharing nothing with tests/gang_preempt_fast.cpp but the rules:

- any node: one pf_preempt call per gang on the state the committed gangs left; the gang commits when every ALLOC member is PLACED;
- one node: one pf_preempt call per node over its [lo, hi) range, the node's cost taken from the evict rows;
- distinct nodes: one call per member, the nodes earlier members use masked as fully pinned in a copy of the bytes.

Also the known-answer cases of tests/golden/kat_gang_preempt.json and the random clusters the CPU and GPU tests share.
"""
from __future__ import annotations

import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import preempt_fast as PF

KAT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_preempt.json")
QUIRKS = {"REF_EXACT": E.QUIRKS_REF_EXACT, "FIXED": E.QUIRKS_FIXED}
POLICY = {"FIRST_FIT": E.POLICY_FIRST_FIT, "BEST_FIT": E.POLICY_BEST_FIT, "RIGHT_TO_LEFT": E.POLICY_RIGHT_TO_LEFT,
          "MIN_FRAG": E.POLICY_MIN_FRAG}
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "NOOP": E.ST_NOOP,
          "GANG_ABORTED": E.ST_GANG_ABORTED}
PER_GANG = 4
LOCALITY = {"ANY": E.GANG_ANY_NODES, "ONE": E.GANG_ONE_NODE, "DISTINCT": E.GANG_DISTINCT_NODES, "PER_GANG": PER_GANG}


def gang_bounds(requests):
    """P1: the [r0, r1) of every maximal run of equal handles."""
    h = np.asarray(requests["handle"])
    starts = [0] + [i for i in range(1, len(h)) if h[i] != h[i - 1]]
    return list(zip(starts, starts[1:] + [len(h)]))


def _span(start, size):
    return ((1 << size) - 1) << start


def _ranked_allocs(req, r0, r1):
    return [r for r in range(r0, r1) if req[r]["op"] == E.OP_ALLOC]


def preempt(node_off, rows, occ, requests, priority, victims, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
            lo=0, hi=None, locality=0):
    """(rc, results, evict) as gang_preempt_fast.preempt returns them, built from pf_preempt calls only."""
    node_off = np.asarray(node_off, dtype=np.uint32)
    rows2 = np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1])
    n_prof = rows2.shape[1]
    G = int(node_off[-1])
    hi = G if hi is None else hi
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    prio = np.ascontiguousarray(priority, dtype=np.uint8)
    vic = np.ascontiguousarray(victims, dtype=E.VICTIM_DTYPE)
    n = len(req)
    dsize = PF.default_sizes(node_off, rows2, node_table)
    if (req["op"] == E.OP_FREE).any():
        return E.EINVAL, None, None
    gangs = gang_bounds(req) if n else []
    locs = []
    for r0, r1 in gangs:                                         # P1 checks
        al = _ranked_allocs(req, r0, r1)
        if len({int(prio[r]) for r in al}) > 1:
            return E.EINVAL, None, None
        if locality == PER_GANG:
            b = [int(req[r]["start"]) for r in al]
            if len(set(b)) > 1 or any(x == E.GANG_FEW_NODES or x > E.GANG_DISTINCT_NODES for x in b):
                return E.EINVAL, None, None
            locs.append(int(req[al[0]]["start"]) if al else 0)
        else:
            locs.append(locality)
    rc, _, _ = PF.preempt(node_off, rows2, occ, req[:0], prio[:0], vic, quirks=quirks, policy=policy, node_table=node_table, lo=lo, hi=hi)
    if rc != E.OK:                                               # rule 2's victim checks
        return rc, None, None
    occ = np.array(occ, dtype=np.uint8)
    alive = np.ones(len(vic), dtype=bool)
    out = np.zeros(n, dtype=E.RESULT_DTYPE)
    evict = np.full((n, 8), E.GPU_NONE, dtype=np.uint32)
    for i in range(n):
        op, p = int(req[i]["op"]), int(req[i]["profile"])
        out[i] = ((E.GPU_NONE, 9, 0, E.ST_NOOP) if op != E.OP_ALLOC else (E.GPU_NONE, 9, 0, E.ST_BAD_PROFILE) if p >= n_prof
                  else (E.GPU_NONE, 9, int(dsize[p]), E.ST_NO_CAPACITY))
    descending = policy == E.POLICY_RIGHT_TO_LEFT

    def call(sub, occ_view, alive_view, a, b):
        idx = np.flatnonzero(alive_view)
        rc, o, ev = PF.preempt(node_off, rows2, occ_view, req[sub], prio[sub], vic[idx], quirks=quirks, policy=policy,
                               node_table=node_table, lo=a, hi=b)
        assert rc == E.OK
        if len(idx):
            ev = np.where(ev == E.GPU_NONE, E.GPU_NONE, idx[np.minimum(ev, len(idx) - 1)]).astype(np.uint32)
        return o, ev

    def commit(rs, o, ev):
        for r, rec, row in zip(rs, o, ev):
            out[r] = rec
            evict[r] = row
            if rec["status"] != E.ST_PLACED:
                continue
            for k in row[row != E.GPU_NONE]:
                alive[k] = False
                occ[vic[k]["gpu"]] &= ~_span(int(vic[k]["start"]), int(vic[k]["size"])) & 0xFF
            occ[rec["gpu"]] |= _span(int(rec["start"]), int(rec["size"]))

    def abort(r0, r1, keep_rank):
        for rank, r in enumerate(_ranked_allocs(req, r0, r1)):
            if rank != keep_rank:
                p = int(req[r]["profile"])
                out[r] = (E.GPU_NONE, 9, int(dsize[p]) if p < n_prof else 0, E.ST_GANG_ABORTED)
                evict[r] = E.GPU_NONE

    def node_of(g):
        return int(np.searchsorted(node_off, g, side="right")) - 1

    for (r0, r1), loc in zip(gangs, locs):
        al = _ranked_allocs(req, r0, r1)
        if not al:
            continue
        if loc == E.GANG_ANY_NODES:
            o, ev = call(al, occ, alive, lo, hi)
            bad = [k for k, rec in enumerate(o) if rec["status"] != E.ST_PLACED]
            if bad:
                abort(r0, r1, bad[0])
            else:
                commit(al, o, ev)
        elif loc == E.GANG_DISTINCT_NODES:
            used, placed, failed = [], [], None
            occ0, alive0 = occ.copy(), alive.copy()
            for rank, r in enumerate(al):
                occ_m, alive_m = occ.copy(), alive.copy()
                for j in used:
                    occ_m[node_off[j]:node_off[j + 1]] = 0xFF
                    alive_m &= ~((vic["gpu"] >= node_off[j]) & (vic["gpu"] < node_off[j + 1]))
                o, ev = call([r], occ_m, alive_m, lo, hi)
                if o[0]["status"] != E.ST_PLACED:
                    failed = rank
                    break
                commit([r], o, ev)
                placed.append(r)
                used.append(node_of(int(o[0]["gpu"])))
            if failed is not None:
                occ[:], alive[:] = occ0, alive0
                abort(r0, r1, failed)
        else:                                                    # one node
            js = np.arange(node_of(lo), node_of(hi - 1) + 1)
            js = js[np.minimum(node_off[js + 1], hi) > np.maximum(node_off[js], lo)]     # an empty node takes nothing
            best, depth = None, 0
            for pos, j in enumerate(js[::-1] if descending else js):
                a, b = max(int(node_off[j]), lo), min(int(node_off[j + 1]), hi)
                o, ev = call(al, occ, alive, a, b)
                placed = [rec["status"] == E.ST_PLACED for rec in o]
                d = placed.index(False) if False in placed else len(al)
                depth = max(depth, d)
                if d == len(al):
                    pr = [int(vic[k]["priority"]) for row in ev for k in row if k != E.GPU_NONE]
                    key = (max(pr) + 1 if pr else 0, sum(pr), len(pr), pos)
                    if best is None or key < best[0]:
                        best = (key, o, ev)
            if best is None:
                abort(r0, r1, depth)
            else:
                commit(al, best[1], best[2])
    return E.OK, out, evict


# ---- known answers ---------------------------------------------------------------------------------------------------------------------
def kat_cases():
    with open(KAT) as f:
        return json.load(f)["cases"]


def case_inputs(case):
    """node_off, rows [n_tables][n_names], node_table, occ, requests, priorities, victims, quirks, policy, lo, hi, locality of a case.
    A request is [handle, profile name or "NOOP", priority, start byte]."""
    names, rows = E.make_profile_tables([tables.TABLES[t] for t in case["tables"]])
    req = np.zeros(len(case["requests"]), dtype=E.REQUEST_DTYPE)
    for i, (h, p, _r, b) in enumerate(case["requests"]):
        req[i]["handle"] = h
        req[i]["op"] = E.OP_NOOP if p == "NOOP" else E.OP_ALLOC
        req[i]["profile"] = 0 if p == "NOOP" else names.index(p) if p in names else E.PROFILE_UNKNOWN
        req[i]["start"] = b
    prio = np.array([r for _h, _p, r, _b in case["requests"]], dtype=np.uint8)
    vic = np.zeros(len(case["victims"]), dtype=E.VICTIM_DTYPE)
    for k, (g, s, z, r) in enumerate(case["victims"]):
        vic[k] = (g, s, z, r, 0)
    node_off = np.array(case["node_off"], dtype=np.uint32)
    return (node_off, rows, np.array(case["node_table"], dtype=np.uint8), np.array(case["occ"], dtype=np.uint8), req, prio, vic,
            QUIRKS[case["quirks"]], POLICY[case["policy"]], case.get("lo", 0), case.get("hi", int(node_off[-1])),
            LOCALITY[case["locality"]])


def expected(case):
    recs = [(E.GPU_NONE if g is None else g, s, z, STATUS[st]) for g, s, z, st in case["records"]]
    return recs, [list(e) for e in case["evict"]]


# ---- random clusters -------------------------------------------------------------------------------------------------------------------
def random_rows(rnd, n_tables=None):
    """[n_tables][n_names] rows of 1..3 reference tables."""
    while True:                                                  # an engine loads at most 16 profile names
        picked = rnd.sample(list(tables.TABLES), n_tables or rnd.randint(1, 3))
        names, rows = E.make_profile_tables([tables.TABLES[t] for t in picked])
        if len(names) <= E.MAX_PROFILES:
            return names, rows


def random_case(rnd, n_gpus, n_req, rows, max_gang=4, locality=None, policy=None, quirks=None, partition=True, victim_share=0.8):
    """A random cluster, victim list and gang burst: (inputs as case_inputs returns them).  Node cuts are random; every busy span is
    split into runs of 1..4 slices, most of them listed as victims at random priorities (255 included)."""
    n_tables, n_prof = rows.shape[0], rows.shape[1]
    n_nodes = rnd.randint(1, max(1, min(n_gpus, 12)))
    cuts = sorted(rnd.sample(range(1, n_gpus), n_nodes - 1)) if n_nodes > 1 else []
    node_off = np.array([0] + cuts + [n_gpus], dtype=np.uint32)
    node_table = np.array([rnd.randrange(n_tables) for _ in range(n_nodes)], dtype=np.uint8)
    occ = np.zeros(n_gpus, dtype=np.uint8)
    vic = []
    for g in range(n_gpus):
        s = 0
        while s < 8:
            z = rnd.randint(1, 4)
            z = min(z, 8 - s)
            if rnd.random() < 0.55:
                occ[g] |= ((1 << z) - 1) << s
                if rnd.random() < victim_share:
                    vic.append((g, s, z, rnd.choice([0, 1, 2, 3, 5, 9, 100, 200, 254, 255])))
            s += z
    rnd.shuffle(vic)
    victims = np.zeros(len(vic), dtype=E.VICTIM_DTYPE)
    for k, (g, s, z, r) in enumerate(vic):
        victims[k] = (g, s, z, r, 0)
    locality = rnd.choice([0, 1, 3, PER_GANG]) if locality is None else locality
    req = np.zeros(n_req, dtype=E.REQUEST_DTYPE)
    prio = np.zeros(n_req, dtype=np.uint8)
    i, h = 0, 0
    while i < n_req:
        k = min(n_req - i, rnd.randint(1, max_gang))
        pr = rnd.choice([0, 1, 3, 6, 50, 150, 255])
        lb = rnd.choice([0, 1, 3])
        for r in range(i, i + k):
            req[r]["handle"] = h
            u = rnd.random()
            req[r]["op"] = E.OP_NOOP if u < 0.06 else E.OP_ALLOC
            req[r]["profile"] = E.PROFILE_UNKNOWN if u > 0.98 else rnd.randrange(n_prof)
            req[r]["start"] = lb if locality == PER_GANG else rnd.randrange(9)
            req[r]["size"] = rnd.randrange(9)
            prio[r] = pr
        i += k
        h += rnd.randint(1, 3)
    lo, hi = 0, n_gpus
    if partition and rnd.random() < 0.3 and n_gpus > 1:
        lo = rnd.randrange(n_gpus)
        hi = rnd.randint(lo + 1, n_gpus)
    policy = rnd.choice([E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]) if policy is None else policy
    quirks = rnd.choice([E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED]) if quirks is None else quirks
    return node_off, rows, node_table, occ, req, prio, victims, quirks, policy, lo, hi, locality


def node_index_case(policy=E.POLICY_FIRST_FIT):
    """A one-node gang of two 1g.5gb on three GPUs whose partition touches 2^20 + 2 node indices: node 0 (GPU 0) is pinned full, node 1
    (GPU 1) has one free slice, 2^20 - 1 empty nodes follow, and node 2^20 + 1 (GPU 2) is free and takes the gang.  2^20 + 1 = 1 modulo
    2^20: a node field of 20 bits would name node 1."""
    names, rows = E.make_profile_tables([tables.A100_40GB])
    node_off = np.concatenate([[0, 1, 2], np.full((1 << 20) - 1, 2), [3]]).astype(np.uint32)
    occ = np.array([0xFF, 0xFE, 0x00], dtype=np.uint8)
    req = np.zeros(2, dtype=E.REQUEST_DTYPE)
    req["profile"] = names.index("1g.5gb")
    return (node_off, rows, None, occ, req, np.ones(2, dtype=np.uint8), np.zeros(0, dtype=E.VICTIM_DTYPE), E.QUIRKS_REF_EXACT, policy,
            0, 3, E.GANG_ONE_NODE)


def run(checker, inputs):
    node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc = inputs
    return checker(node_off, rows, occ, req, prio, vic, quirks=quirks, policy=policy, node_table=node_table, lo=lo, hi=hi, locality=loc)
