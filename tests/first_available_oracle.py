"""Second restatement of profile alternatives (ISL_FLAG_FIRST_AVAILABLE, include/islplace.h A1-A8), built on the unchanged checkers of
isl_place_batch one alternative at a time, plus the known-answer vectors.

It shares nothing with tests/first_available_fast.cpp but the rules: the FREEs go through one checker call with every ALLOC made a NOOP
(A2), then every alternative of every pod is one single-request call on the occupancy the calls before it left (A3), through
``range_oracle.place_range`` for FIRST_FIT and RIGHT_TO_LEFT, ``bestfit_fast.place`` for BEST_FIT and MIN_FRAG and
``node_score_fast.place`` for MOST_ / LEAST_ALLOCATED.  An alternative after the placed one of its pod is never looked at: it gets the
default record with status ALT_SKIPPED.
"""
from __future__ import annotations

import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import bestfit_fast as BF
import node_score_fast as NF
import range_oracle as RO
from preempt_fast import default_sizes

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_first_available.json")
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "FREED": E.ST_FREED,
          "BAD_SPAN": E.ST_BAD_SPAN, "NOOP": E.ST_NOOP, "ALT_SKIPPED": E.ST_ALT_SKIPPED}
QUIRKS = {"REF_EXACT": E.QUIRKS_REF_EXACT, "FIXED": E.QUIRKS_FIXED}
POLICY = {"FIRST_FIT": E.POLICY_FIRST_FIT, "BEST_FIT": E.POLICY_BEST_FIT, "RIGHT_TO_LEFT": E.POLICY_RIGHT_TO_LEFT,
          "MIN_FRAG": E.POLICY_MIN_FRAG, "MOST_ALLOCATED": E.POLICY_MOST_ALLOCATED, "LEAST_ALLOCATED": E.POLICY_LEAST_ALLOCATED}


def _checker(node_off, rows, occ, requests, policy, quirks, node_table, lo, hi):
    """isl_place_batch_range(lo, hi, requests) on an unflagged engine: (records, occupancy after)."""
    if policy in (E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT):
        return RO.place_range(node_off, rows, occ, lo, hi, requests, quirks, policy, node_table)
    if policy in (E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG):
        return BF.place(node_off, rows, occ, requests, quirks, policy, node_table, lo, hi)
    return NF.place(node_off, rows, occ, requests, policy, quirks, node_table, lo, hi)


def pod_starts(requests):
    """A1: True where an ALLOC opens a pod (the request before it is no ALLOC or has another handle), False elsewhere."""
    req = np.asarray(requests, dtype=E.REQUEST_DTYPE)
    alloc = req["op"] == E.OP_ALLOC
    cont = np.zeros(len(req), dtype=bool)
    cont[1:] = alloc[1:] & alloc[:-1] & (req["handle"][1:] == req["handle"][:-1])
    return alloc & ~cont


def place(node_off, rows, occ, requests, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0, hi=None):
    """One batch on an ISL_FLAG_FIRST_AVAILABLE engine: (records, occupancy after, placed pods)."""
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    hi = int(np.asarray(node_off)[-1]) if hi is None else hi
    frees = req.copy()
    frees["op"][req["op"] == E.OP_ALLOC] = E.OP_NOOP
    out, occ = _checker(node_off, rows, occ, frees, policy, quirks, node_table, lo, hi)
    dsize = default_sizes(node_off, rows, node_table)
    opens = pod_starts(req)
    done, placed = False, 0
    for i in np.flatnonzero(req["op"] == E.OP_ALLOC):
        if opens[i]:
            done = False
        p = int(req["profile"][i])
        if done:
            out[i] = (E.GPU_NONE, E.START_NONE, dsize[p] if p < len(dsize) else 0, E.ST_ALT_SKIPPED)
            continue
        rec, after = _checker(node_off, rows, occ, req[i:i + 1], policy, quirks, node_table, lo, hi)
        out[i] = rec[0]
        if rec[0]["status"] == E.ST_PLACED:
            occ, done = after, True
            placed += 1
    return out, occ, placed


def chosen_only(requests, records):
    """A5 (b): the requests with every alternative but each pod's PLACED one turned into a NOOP."""
    req = np.array(requests, dtype=E.REQUEST_DTYPE)
    drop = (req["op"] == E.OP_ALLOC) & (np.asarray(records)["status"] != E.ST_PLACED)
    req["op"][drop] = E.OP_NOOP
    return req


# ---- known-answer vectors ---------------------------------------------------------------------------------------------------------
def kat_cases():
    with open(KAT_PATH) as f:
        return json.load(f)["cases"]


def runs(rle):
    return np.array([b for b, k in rle for _ in range(k)], dtype=np.uint8)


def case_inputs(case):
    """node_off, rows [n_tables][n_names], node_table, occ, requests, quirks, policy, (lo, hi) of a known-answer case."""
    names, rows = E.make_profile_tables([tables.TABLES[t] for t in case["tables"]])
    req = np.zeros(len(case["requests"]), dtype=E.REQUEST_DTYPE)
    for i, r in enumerate(case["requests"]):
        if r[0] == "alloc":             # ["alloc", name, handle]
            req[i] = (r[2], names.index(r[1]) if r[1] in names else E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
        elif r[0] == "free":            # ["free", gpu, start, size]
            req[i] = (r[1], 0, E.OP_FREE, r[2], r[3])
        else:                           # ["noop", handle]
            req[i] = (r[1], 0, E.OP_NOOP, 0, 0)
    node_off = np.array(case["node_off"], dtype=np.uint32)
    lo, hi = case.get("range", (0, int(node_off[-1])))
    return (node_off, rows, np.array(case["node_table"], dtype=np.uint8), runs(case["occ"]), req, QUIRKS[case["quirks"]],
            POLICY[case["policy"]], (lo, hi))


def expected(case):
    return [(E.GPU_NONE if g is None else g, s, z, STATUS[st]) for g, s, z, st in case["records"]]


def as_tuples(records):
    return [tuple(int(x) for x in r) for r in records]
