"""Second restatement of isl_preempt (include/islplace.h, rules 1-6), on CR-shaped dicts, plus the known-answer vectors.

It shares nothing with tests/preempt_fast.cpp but the rules: GPUs come from the Instaslice objects (nodes in list order, GPUs by sorted
UUID), each node's own Migplacement gives the rows (first row of a name), every busy slice comes from a dangling Prepared entry or an
Allocations entry, and only allocations of the caller's victim set may leave.  Priorities here are already ranks (0..255).
"""
from __future__ import annotations

import json
import os

from instaslice_b200 import engine as E
from instaslice_b200 import tables

KAT_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_preempt.json")
STATUS = {"PLACED": E.ST_PLACED, "NO_CAPACITY": E.ST_NO_CAPACITY, "BAD_PROFILE": E.ST_BAD_PROFILE, "NOOP": E.ST_NOOP}
QUIRKS = {"REF_EXACT": E.QUIRKS_REF_EXACT, "FIXED": E.QUIRKS_FIXED}
POLICY = {"FIRST_FIT": E.POLICY_FIRST_FIT, "BEST_FIT": E.POLICY_BEST_FIT, "RIGHT_TO_LEFT": E.POLICY_RIGHT_TO_LEFT,
          "MIN_FRAG": E.POLICY_MIN_FRAG}


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


def preempt_cr(items, pods, victim_rank, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT):
    """``pods``: [{"profile", "rank"}]; ``victim_rank``: {allocation pod UID: rank} of the allocations that may leave.

    Returns per pod ("fits" | "preempt" | "none", {"nodename", "gpuUUID", "start", "size"} or None, [victim UIDs by start])."""
    gpus = [(it["metadata"]["name"], u, it) for it in items for u in sorted(it["spec"]["MigGPUUUID"])]
    if policy == E.POLICY_RIGHT_TO_LEFT:
        gpus = gpus[::-1]
    # per GPU: 8 slots, each None (free), "pinned" or the UID of the victim that covers it
    slots = []
    for _node, uuid, it in gpus:
        s = [None] * 8
        spec = it["spec"]
        busy = [("pinned", p) for p in spec.get("prepared", {}).values() if p["parent"] == uuid and p.get("podUUID", "") == ""]
        busy += [(uid if uid in victim_rank else "pinned", a) for uid, a in spec.get("allocations", {}).items() if a["gpuUUID"] == uuid]
        for who, x in busy:
            for k in range(int(x["start"]), int(x["start"]) + int(x["size"])):
                s[k] = who
        slots.append(s)
    starts_of = {}                      # (node, name) -> (size, starts) of the node's first row with the name
    for it in items:
        for row in reversed(it["spec"].get("migplacement", [])):
            starts_of[(it["metadata"]["name"], row["profile"])] = (row["placements"][0]["size"], [p["start"] for p in row["placements"]])
    out = []
    for pod in pods:
        best = None
        for pos, (node, uuid, _it) in enumerate(gpus):
            row = starts_of.get((node, pod["profile"]))
            if row is None:
                continue
            size, starts = row
            for k, v in enumerate(starts):
                if not legal(size, v, quirks):
                    continue
                gone = {slots[pos][x] for x in range(v, v + size) if slots[pos][x] is not None}
                if "pinned" in gone or any(victim_rank[u] >= pod["rank"] for u in gone):
                    continue
                ranks = [victim_rank[u] for u in gone]
                key = (max(ranks) + 1 if ranks else 0, sum(ranks), len(ranks), pos, k)
                if best is None or key < best[0]:
                    best = (key, pos, v, size, gone)
        if best is None:
            out.append(("none", None, []))
            continue
        _key, pos, v, size, gone = best
        s = slots[pos]
        order = sorted(gone, key=lambda u: s.index(u))
        for x in range(8):
            if s[x] in gone:
                s[x] = None
        for x in range(v, v + size):
            s[x] = "pinned"
        node, uuid, _it = gpus[pos]
        where = {"nodename": node, "gpuUUID": uuid, "start": v, "size": size}
        out.append(("preempt", where, order) if order else ("fits", where, []))
    return out


def case_items(case):
    """The Instaslice objects of a known-answer case: one node per node_off entry, GPUs named so that sorted UUID = canonical order,
    victims as allocations "v<index>", every other busy slice as dangling Prepared slices."""
    node_off, occ = case["node_off"], case["occ"]
    items = []
    for n in range(len(node_off) - 1):
        mig = tables.migplacement(tables.TABLES[case["tables"][case["node_table"][n]]])
        items.append({"metadata": {"name": "node-%d" % n},
                      "spec": {"MigGPUUUID": {"GPU-%06d" % g: "" for g in range(node_off[n], node_off[n + 1])}, "migplacement": mig,
                               "prepared": {}, "allocations": {}}})
    covered = [0] * len(occ)
    for k, (g, start, size, _prio) in enumerate(case["victims"]):
        n = max(i for i in range(len(node_off) - 1) if node_off[i] <= g)
        items[n]["spec"]["allocations"]["v%d" % k] = {"gpuUUID": "GPU-%06d" % g, "start": start, "size": size, "allocationStatus": "created"}
        covered[g] |= span(start, size)
    for g, b in enumerate(occ):
        n = max(i for i in range(len(node_off) - 1) if node_off[i] <= g)
        rest = b & ~covered[g]
        for x in range(8):
            if rest >> x & 1:
                items[n]["spec"]["prepared"]["p%d-%d" % (g, x)] = {"parent": "GPU-%06d" % g, "start": x, "size": 1, "podUUID": ""}
    return items


def expected(case):
    """(records as tuples with GPU_NONE for null, evict lists) of a case."""
    recs = [(E.GPU_NONE if g is None else g, s, z, STATUS[st]) for g, s, z, st in case["records"]]
    return recs, [list(e) for e in case["evict"]]


def case_inputs(case):
    """The engine's inputs of a case: node_off, rows [n_tables][n_names], node_table, occ, requests, priorities, victims, quirks, policy."""
    import numpy as np

    names, rows = E.make_profile_tables([tables.TABLES[t] for t in case["tables"]])
    req = np.zeros(len(case["requests"]), dtype=E.REQUEST_DTYPE)
    req["handle"] = np.arange(len(req))
    req["profile"] = [names.index(p) if p in names else E.PROFILE_UNKNOWN for p, _ in case["requests"]]
    req["op"] = E.OP_ALLOC
    prio = np.array([r for _, r in case["requests"]], dtype=np.uint8)
    vic = np.zeros(len(case["victims"]), dtype=E.VICTIM_DTYPE)
    for k, (g, s, z, r) in enumerate(case["victims"]):
        vic[k] = (g, s, z, r, 0)
    return (np.array(case["node_off"], dtype=np.uint32), rows, np.array(case["node_table"], dtype=np.uint8),
            np.array(case["occ"], dtype=np.uint8), req, prio, vic, QUIRKS[case["quirks"]], POLICY[case["policy"]])
