"""CPU restatements of isl_place_gangs on an engine created with ISL_FLAG_GANG_MIN_MEMBERS (TEST INFRASTRUCTURE, NOT PRODUCT CODE):
elastic gangs, built by truncation (include/islplace.h M5 b) on the existing checkers, which stay unchanged.  A gang is run whole by the
checker of its locality; when it aborts at ALLOC member f (the one whose record is not GANG_ABORTED) and f >= m', the gang cut to its
first f ALLOC members is run again from the same occupancy, and it must commit.  Two compositions that share nothing with each other,
or with tests/gang_min_fast.cpp, but M3:

``fast_gangs_min``     every policy: the call's FREEs, then each gang alone through ``gang_locality_oracle.fast_gangs_locality`` (the
                       brute force of its locality), with the occupancy carried from one gang to the next.  Returns the records, the
                       occupancy after the call and the members placed.
``ref_py_gangs_min``   first-fit on CR-shaped dicts: each gang through ``gang_locality_oracle.ref_py_gangs_locality``.
``load_kat``           the hand-worked vectors of tests/golden/kat_gang_min.json as engine inputs.
"""
from __future__ import annotations

import copy
import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import gang_few_oracle as GFO
import gang_locality_oracle as GLO
from gang_min_fast import effective_minimum

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_min.json")
STATUS = dict(GLO.STATUS, TRIMMED=E.ST_GANG_TRIMMED)
FLAG_OF = GLO.FLAG_OF


def with_minimum(requests, gang_off, min_members) -> np.ndarray:
    """A copy of ``requests`` whose ALLOC members carry their gang's minimum in ``size`` (what ``Engine.place_gangs`` writes)."""
    req = np.array(requests, dtype=E.REQUEST_DTYPE)
    per = np.repeat(np.asarray(min_members, dtype=np.int64), np.diff(np.asarray(gang_off, dtype=np.int64)))
    alloc = req["op"] == E.OP_ALLOC
    req["size"][alloc] = per[alloc].astype(np.uint8)
    return req


def fast_gangs_min(node_off, rows, occ, requests, gang_off, locality, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT,
                   node_table=None, lo=0, hi=None):
    """``locality``: one ``E.GANG_*`` per gang; the minima are the ALLOC members' ``size`` bytes (M1)."""
    node_off = np.asarray(node_off, dtype=np.uint32)
    hi = int(node_off[-1]) if hi is None else hi
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.asarray(gang_off, dtype=np.int64)
    mins = effective_minimum(req, gang_off)
    alloc = req["op"] == E.OP_ALLOC
    rest = req.copy()
    rest["op"][alloc] = E.OP_NOOP
    out, cur = GLO.fast_gangs_locality(node_off, rows, occ, rest, [0, len(req)], quirks, policy, node_table, lo, hi)    # FREEs first
    placed = 0

    def alone(members, loc, occ_in):
        members = members.copy()
        members["start"], members["size"] = 0, 0
        return GLO.fast_gangs_locality(node_off, rows, occ_in, GLO.with_locality(members, [0, len(members)], [loc]), [0, len(members)],
                                       quirks, policy, node_table, lo, hi)

    for g, (a, b) in enumerate(zip(gang_off[:-1], gang_off[1:])):
        idx = np.flatnonzero(alloc[a:b]) + a
        if not len(idx):
            continue
        got, after = alone(req[idx], int(locality[g]), cur)
        if (got["status"] == E.ST_PLACED).all():
            out[idx], cur = got, after
            placed += len(idx)
            continue
        f = int(np.flatnonzero(got["status"] != E.ST_GANG_ABORTED)[0])
        out[idx] = got                                  # M4, or member f's record and the unplaced records for M3
        if f >= int(mins[g]):                           # M3: the cut gang commits where the run put it
            cut, cur = alone(req[idx[:f]], int(locality[g]), cur)
            assert (cut["status"] == E.ST_PLACED).all(), "a gang cut at the member it failed at must commit"
            out[idx[:f]] = cut
            out["status"][idx[f + 1:]] = E.ST_GANG_TRIMMED
            placed += f
    return out, np.asarray(cur, dtype=np.uint8), placed


def ref_py_gangs_min(crs: list, gangs: list, locality: list, min_members: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``, one locality and one minimum m (0..255) per gang; ``crs`` one Instaslice dict per
    node, updated in place.  Returns per gang ("placed", [AllocationDetails...]), ("trimmed", [AllocationDetails of the first f], f) or
    ("aborted", index of the member that keeps its record)."""
    out = []
    for gang, loc, m in zip(gangs, locality, min_members):
        need = len(gang) if m == 0 or m >= len(gang) else m
        before = copy.deepcopy(crs)
        verdict = GLO.ref_py_gangs_locality(crs, [gang], [loc], quirks)[0]
        if verdict[0] == "aborted" and verdict[1] >= need:
            crs[:] = before
            cut = GLO.ref_py_gangs_locality(crs, [gang[:verdict[1]]], [loc], quirks)[0]
            assert cut[0] == "placed", "a gang cut at the member it failed at must commit"
            verdict = ("trimmed", cut[1], verdict[1])
        out.append(verdict)
    return out


def kat_requests(gangs, names):
    """Requests and gang offsets of one vector: a member is a profile name, ["FREE", gpu, start, size] or ["NOOP", size byte]."""
    req = np.zeros(sum(len(g) for g in gangs), dtype=E.REQUEST_DTYPE)
    i = 0
    for g in gangs:
        for m in g:
            if isinstance(m, list) and m[0] == "NOOP":
                req[i] = (i, 0, E.OP_NOOP, 0, m[1])
            elif isinstance(m, list):
                req[i] = (m[1], 0, E.OP_FREE, m[2], m[3])
            else:
                req[i] = (i, names.index(m) if m in names else E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
            i += 1
    return req, np.cumsum([0] + [len(g) for g in gangs]).astype(np.uint32)


def load_kat():
    """Yield per vector: (name, engine inputs dict, requests with their localities and minima, gang offsets, expected records, expected
    occupancy, expected members placed)."""
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
        req = with_minimum(GLO.with_locality(req, off, v["locality"]), off, v["min_members"])
        want = [(E.GPU_NONE if r[0] is None else r[0], r[1], r[2], STATUS[r[3]]) for g in v["records"] for r in g]
        inputs = {"node_off": np.asarray(v["node_off"], dtype=np.uint32), "rows": rows, "occ": np.asarray(v["occ"], dtype=np.uint8),
                  "policy": GFO.POLICY[v["policy"]], "quirks": E.QUIRKS_REF_EXACT if v["quirks"] == "ref_exact" else E.QUIRKS_FIXED,
                  "node_table": None if v.get("node_table") is None else np.asarray(v["node_table"], dtype=np.uint8),
                  "partition": v.get("partition"), "table_names": v["tables"], "names": names, "gangs": v["gangs"],
                  "locality": v["locality"], "min_members": v["min_members"]}
        yield v["name"], inputs, req, off, want, np.asarray(v["occ_after"], dtype=np.uint8), v["placed"]
