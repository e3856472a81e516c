"""CPU restatements of balanced gangs (isl_place_gangs on an ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_BALANCED engine; TEST
INFRASTRUCTURE, NOT PRODUCT CODE) that share nothing with tests/gang_balance_fast.cpp beyond the rules of include/islplace.h (B1-B8):

``fast_gangs_balance``      every policy and locality byte: the call's FREEs, then gang after gang on the occupancy the earlier ones
                            left (L2).  A byte of 0..3 goes to ``gang_locality_oracle.fast_gangs_locality``; a balanced gang is placed
                            member by member: every node of the range with a GPU that admits the member proposes its own choice (a
                            ``RangeFast`` over that node's GPUs), mu is the least count among the proposing nodes, and the proposals of
                            the nodes within the skew are compared by (policy score, scan position).  ``elastic``: a gang that stops at
                            ALLOC member f >= m' commits its first f members (M3, B5).  Returns the records, the occupancy after the
                            call and the members placed.
``ref_py_gangs_balance``    first-fit on CR-shaped dicts: per member ``ref_py.find_device_for_a_slice`` tells which nodes admit it, and
                            ``ref_py.reconcile_gated_pod`` runs the reference's node loop over the nodes within the skew of a deep
                            copy of the cluster; a gang whose members all come back "placed" replaces the cluster with the copy.
``load_kat``                the hand-worked vectors of tests/golden/kat_gang_balance.json as engine inputs.
"""
from __future__ import annotations

import copy
import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables
from oracle import ref_py

import gang_locality_oracle as GLO
from gang_min_fast import effective_minimum
from gang_oracle import default_sizes
from gang_spread_oracle import POLICY, _score
from range_oracle import RangeFast

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_gang_balance.json")
STATUS = dict(GLO.STATUS, TRIMMED=E.ST_GANG_TRIMMED)


def _balanced_gang(node_off, rows, cur, members, skew, quirks, policy, table, per_node, lo, hi):
    """The ALLOC ``members`` of one balanced gang on occupancy ``cur``: (their records as far as they placed, occupancy with them)."""
    n_nodes, G = len(node_off) - 1, int(node_off[-1])
    tent, cnt, got = np.array(cur, dtype=np.uint8), [0] * n_nodes, []
    for i in range(len(members)):
        if int(members["profile"][i]) >= rows.shape[-1]:
            break
        props = []                                      # (count, (score, scan position), record, node) per admitting node
        for n in range(n_nodes):
            nlo, nhi = max(int(node_off[n]), lo), min(int(node_off[n + 1]), hi)
            if nlo >= nhi:
                continue
            r = RangeFast(node_off, rows, tent, nlo, nhi, quirks, policy, node_table=per_node).place(members[i:i + 1])[0]
            if r["status"] != E.ST_PLACED:
                continue
            g, mine = int(r["gpu"]), ((1 << int(r["size"])) - 1) << int(r["start"])
            key = (_score(policy, rows[table[n]] if rows.ndim == 2 else rows, quirks, int(tent[g]), mine),
                   G - 1 - g if policy == E.POLICY_RIGHT_TO_LEFT else g)
            props.append((cnt[n], key, r, n))
        if not props:
            break
        mu = min(p[0] for p in props)
        _c, _key, r, n = min((p for p in props if p[0] <= mu + skew - 1), key=lambda p: p[1])
        tent[int(r["gpu"])] |= ((1 << int(r["size"])) - 1) << int(r["start"])
        cnt[n] += 1
        got.append(r)
    return got, tent


def fast_gangs_balance(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
                       lo=0, hi=None, elastic=False):
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
    out, cur = GLO.fast_gangs_locality(node_off, rows, occ, rest, [0, len(req)], quirks, policy, node_table, lo, hi)    # FREEs first
    mins = effective_minimum(req, gang_off) if elastic else None
    placed = 0

    def alone(members, loc, occ_in):
        """One gang's ALLOC members by its locality: records as isl_place_gangs writes them, occupancy after (that before on abort)."""
        if loc <= E.GANG_DISTINCT_NODES:
            return GLO.fast_gangs_locality(node_off, rows, occ_in, members, [0, len(members)], quirks, policy, node_table, lo, hi)
        got, tent = _balanced_gang(node_off, rows, occ_in, members, loc - E.GANG_DISTINCT_NODES, quirks, policy, table, per_node, lo, hi)
        if len(got) == len(members):
            return np.array(got, dtype=E.RESULT_DTYPE), tent
        res = np.zeros(len(members), dtype=E.RESULT_DTYPE)
        for k, p in enumerate(members["profile"].astype(np.int64)):
            known = p < rows.shape[-1]
            res[k] = (E.GPU_NONE, E.START_NONE, sizes[p] if known else 0,
                      E.ST_GANG_ABORTED if k != len(got) else E.ST_NO_CAPACITY if known else E.ST_BAD_PROFILE)
        return res, np.array(occ_in, dtype=np.uint8)

    for g, (a, b) in enumerate(zip(gang_off[:-1], gang_off[1:])):
        idx = np.flatnonzero(alloc[a:b]) + a
        if not len(idx):
            continue
        loc = int(req["start"][idx[0]])
        got, after = alone(req[idx], loc, cur)
        if (got["status"] == E.ST_PLACED).all():
            out[idx], cur = got, after
            placed += len(idx)
            continue
        f = int(np.flatnonzero(got["status"] != E.ST_GANG_ABORTED)[0])
        out[idx] = got
        if elastic and f >= int(mins[g]):               # M3: the gang cut to its first f members commits where the run put them
            cut, cur = alone(req[idx[:f]], loc, cur)
            assert (cut["status"] == E.ST_PLACED).all(), "a gang cut at the member it failed at must commit"
            out[idx[:f]] = cut
            out["status"][idx[f + 1:]] = E.ST_GANG_TRIMMED
            placed += f
    return out, np.asarray(cur, dtype=np.uint8), placed


def ref_py_gangs_balance(crs: list, gangs: list, skews: list, quirks: int) -> list:
    """``gangs``: lists of ``(pod, profile_name)``, one maxSkew per gang; ``crs`` one Instaslice dict per node, updated in place.
    Returns per gang ("placed", [AllocationDetails...]) or ("aborted", index of the member that found nothing)."""
    out = []
    for gang, skew in zip(gangs, skews):
        shadow = copy.deepcopy(crs)
        cnt, allocs = [0] * len(shadow), []
        for k, (pod, name) in enumerate(gang):
            admits = [n for n, cr in enumerate(shadow) if ref_py.find_device_for_a_slice(copy.deepcopy(cr), name, pod, quirks) is not None]
            if not admits:
                out.append(("aborted", k))
                break
            mu = min(cnt[n] for n in admits)
            visible = [shadow[n] for n in admits if cnt[n] <= mu + skew - 1]
            verdict, placed = ref_py.reconcile_gated_pod(visible, pod, name, quirks)
            assert verdict == "placed"
            cnt[next(n for n, cr in enumerate(shadow) if placed[0]["gpuUUID"] in cr["spec"]["MigGPUUUID"])] += 1
            allocs.append(placed[0])
        else:
            crs[:] = shadow
            out.append(("placed", allocs))
    return out


def load_kat():
    """Yield per vector: (name, engine inputs dict, requests with their locality and minimum bytes, gang offsets, expected records,
    expected occupancy, expected members placed)."""
    with open(KAT_PATH) as f:
        doc = json.load(f)
    for v in doc["vectors"]:
        tabs = [getattr(tables, t) for t in v["tables"]]
        if len(tabs) == 1:
            rows, names = E.make_profiles(tabs[0]), [r[0] for r in tabs[0]]
        else:
            names, rows = E.make_profile_tables(tabs)
            names = list(names)
        req, off = GLO.kat_requests(v["gangs"], names)
        req = GLO.with_locality(req, off, v["locality"])
        if v.get("min_members") is not None:
            per = np.repeat(np.asarray(v["min_members"], dtype=np.int64), np.diff(off.astype(np.int64)))
            req["size"][req["op"] == E.OP_ALLOC] = per[req["op"] == E.OP_ALLOC]
        want = [(E.GPU_NONE if r[0] is None else r[0], r[1], r[2], STATUS[r[3]]) for g in v["records"] for r in g]
        inputs = {"node_off": np.asarray(v["node_off"], dtype=np.uint32), "rows": rows, "occ": np.asarray(v["occ"], dtype=np.uint8),
                  "policy": POLICY[v["policy"]], "quirks": E.QUIRKS_REF_EXACT if v["quirks"] == "ref_exact" else E.QUIRKS_FIXED,
                  "node_table": None if v.get("node_table") is None else np.asarray(v["node_table"], dtype=np.uint8),
                  "partition": v.get("partition"), "table_names": v["tables"], "names": names, "gangs": v["gangs"],
                  "locality": v["locality"], "elastic": v.get("min_members") is not None}
        yield v["name"], inputs, req, off, want, np.asarray(v["occ_after"], dtype=np.uint8), v["placed"]
