"""Second restatement of node scoring (ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED, include/islplace.h rules 1-7), on CR-shaped
dicts, plus the known-answer vectors.

It shares nothing with tests/node_score_fast.cpp but the rules: GPUs come from the Instaslice objects (nodes in list order, GPUs by
sorted UUID), each node's own Migplacement gives its rows (first row of a name) and its width, every busy slice comes from a dangling
Prepared entry or an Allocations entry, and a placement is committed as a new Allocations entry of the node it lands on.
"""
from __future__ import annotations

import json
import os

import numpy as np

from instaslice_b200 import engine as E
from instaslice_b200 import tables

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_node_score.json")
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "FREED": E.ST_FREED,
          "BAD_SPAN": E.ST_BAD_SPAN, "NOOP": E.ST_NOOP}
QUIRKS = {"REF_EXACT": E.QUIRKS_REF_EXACT, "FIXED": E.QUIRKS_FIXED}
POLICY = {"MOST_ALLOCATED": E.POLICY_MOST_ALLOCATED, "LEAST_ALLOCATED": E.POLICY_LEAST_ALLOCATED}


def kat_cases():
    with open(KAT_PATH) as f:
        return json.load(f)["cases"]


def legal(size, v, quirks):
    """Whether the start search (:343-383) can ever return start v for a size-slice profile."""
    if v > 7 or size < 1 or size > 8:
        return False
    if size == 1:
        return True
    if quirks & E.QUIRK_POW2_ONLY and size not in (2, 4, 8):
        return False
    return v + size < 8 if quirks & E.QUIRK_STRICT_BOUND else v + size <= 8


def span(start, size):
    return ((1 << int(size)) - 1) << int(start)


def _busy_mask(spec, uuid):
    m = 0
    for p in spec.get("prepared", {}).values():
        if p["parent"] == uuid and p.get("podUUID", "") == "":
            m |= span(p["start"], p["size"])
    for a in spec.get("allocations", {}).values():
        if a["gpuUUID"] == uuid:
            m |= span(a["start"], a["size"])
    return m


def place_cr(items, pods, policy, quirks=E.QUIRKS_REF_EXACT, lo=0, hi=None, names=None):
    """One batch on the Instaslice objects ``items``, committed into them.  ``pods``: {"op": "alloc", "profile", "uid"} or
    {"op": "free", "uid"} (the allocation that leaves).  [lo, hi): canonical GPU positions the call sees.  ``names``: the profile names
    the engine was loaded with (default: those of the items' tables); any other name is a bad profile.

    Returns one record per pod as (gpu position or None, start, size, status), the engine's records."""
    gpus = [(n, u) for n, it in enumerate(items) for u in sorted(it["spec"]["MigGPUUUID"])]
    hi = len(gpus) if hi is None else hi
    pos_of = {u: k for k, (_n, u) in enumerate(gpus)}
    rows = []                       # per node: name -> (size, starts) of its first row with the name; its width
    for it in items:
        r = {}
        for row in it["spec"].get("migplacement", []):
            r.setdefault(row["profile"], (row["placements"][0]["size"], [p["start"] for p in row["placements"]]))
        width = max((s + z for z, starts in r.values() for s in starts), default=0)
        rows.append((r, width))
    known = set(names) if names is not None else {name for r, _w in rows for name in r}
    out = [None] * len(pods)
    for i, pod in enumerate(pods):  # FREEs first
        if pod["op"] == "free":
            for it in items:
                a = it["spec"]["allocations"].get(pod["uid"])
                if a is not None:
                    if lo <= pos_of[a["gpuUUID"]] < hi:
                        del it["spec"]["allocations"][pod["uid"]]
                    out[i] = (pos_of[a["gpuUUID"]], a["start"], a["size"], E.ST_FREED)
    for i, pod in enumerate(pods):
        if pod["op"] != "alloc":
            continue
        name = pod["profile"]
        if name not in known:
            out[i] = (None, E.START_NONE, 0, E.ST_BAD_PROFILE)
            continue
        best = None                 # (score, node): the first node with the highest score
        for n, it in enumerate(items):
            mine = [k for k in range(lo, hi) if gpus[k][0] == n]
            r, width = rows[n]
            if not mine or name not in r:
                continue
            size, starts = r[name]
            busy_bytes = [_busy_mask(it["spec"], gpus[k][1]) for k in mine]
            fits = [any(legal(size, v, quirks) and not b & span(v, size) for v in starts) for b in busy_bytes]
            if not any(fits):
                continue
            cap = width * len(mine)
            busy = sum(bin(b & ((1 << width) - 1)).count("1") for b in busy_bytes)
            score = 100 * (busy + size) // cap if policy == E.POLICY_MOST_ALLOCATED else 100 * (cap - busy - size) // cap
            if best is None or score > best[0]:
                best = (score, n)
        if best is None:
            dflt = next((rows[n][0][name][0] for n in range(len(items)) if name in rows[n][0]), 0)
            out[i] = (None, E.START_NONE, dflt, E.ST_NO_CAPACITY)
            continue
        n = best[1]
        size, starts = rows[n][0][name]
        for k in range(lo, hi):
            if gpus[k][0] != n:
                continue
            b = _busy_mask(items[n]["spec"], gpus[k][1])
            v = next((v for v in starts if legal(size, v, quirks) and not b & span(v, size)), None)
            if v is None:
                continue
            items[n]["spec"]["allocations"][pod["uid"]] = {"gpuUUID": gpus[k][1], "start": v, "size": size, "allocationStatus": "creating"}
            out[i] = (k, v, size, E.ST_PLACED)
            break
    return out


def occupancy(items):
    return np.array([_busy_mask(it["spec"], u) for it in items for u in sorted(it["spec"]["MigGPUUUID"])], dtype=np.uint8)


def runs(rle):
    return np.array([b for b, k in rle for _ in range(k)], dtype=np.uint8)


def items_from(node_off, occ, table_names, node_table):
    """Instaslice objects of an inventory: one per node, GPUs named so that sorted UUID = canonical order, every busy slice a dangling
    Prepared slice."""
    items = []
    for n in range(len(node_off) - 1):
        mig = tables.migplacement(tables.TABLES[table_names[int(node_table[n])]])
        gs = range(int(node_off[n]), int(node_off[n + 1]))
        prepared = {"p%d-%d" % (g, x): {"parent": "GPU-%07d" % g, "start": x, "size": 1, "podUUID": ""}
                    for g in gs for x in range(8) if int(occ[g]) >> x & 1}
        items.append({"metadata": {"name": "node-%d" % n},
                      "spec": {"MigGPUUUID": {"GPU-%07d" % g: "" for g in gs}, "migplacement": mig, "prepared": prepared, "allocations": {}}})
    return items


def case_inputs(case):
    """The engine's inputs of a known-answer case: node_off, rows [n_tables][n_names], node_table, occ, requests, quirks, policy, (lo, hi)."""
    names, rows = E.make_profile_tables([tables.TABLES[t] for t in case["tables"]])
    req = np.zeros(len(case["requests"]), dtype=E.REQUEST_DTYPE)
    for i, r in enumerate(case["requests"]):
        if r[0] == "alloc":
            req[i] = (i, names.index(r[1]) if r[1] in names else E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
        else:
            req[i] = (r[1], 0, E.OP_FREE, r[2], r[3])
    node_off = np.array(case["node_off"], dtype=np.uint32)
    lo, hi = case.get("range", (0, int(node_off[-1])))
    return (node_off, rows, np.array(case["node_table"], dtype=np.uint8), runs(case["occ"]), req, QUIRKS[case["quirks"]],
            POLICY[case["policy"]], (lo, hi))


def case_pods(case, items):
    """The requests of a case as pods on ``items``: a FREE names the allocation it releases, made an Allocations entry first."""
    gpus = [(n, u) for n, it in enumerate(items) for u in sorted(it["spec"]["MigGPUUUID"])]
    pods = []
    for i, r in enumerate(case["requests"]):
        if r[0] == "alloc":
            pods.append({"op": "alloc", "profile": r[1], "uid": "pod-%d" % i})
            continue
        n, uuid = gpus[r[1]]
        spec = items[n]["spec"]
        for x in range(r[2], r[2] + r[3]):          # the span's dangling Prepared slices become one allocation
            spec["prepared"].pop("p%d-%d" % (r[1], x), None)
        spec["allocations"]["old-%d" % i] = {"gpuUUID": uuid, "start": r[2], "size": r[3], "allocationStatus": "created"}
        pods.append({"op": "free", "uid": "old-%d" % i})
    return pods


def expected(case):
    return [(E.GPU_NONE if g is None else g, s, z, STATUS[st]) for g, s, z, st in case["records"]]


def as_records(recs):
    return [(E.GPU_NONE if g is None else g, s, z, st) for g, s, z, st in recs]
