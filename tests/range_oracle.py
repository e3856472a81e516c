"""CPU restatement of isl_place_batch_range (TEST INFRASTRUCTURE, NOT PRODUCT CODE): the checker of the restricted-range tests.

``RangeFast`` is an ``oracle.Fast`` over the GPUs [lo, hi) of a whole inventory, with the ``.place`` / ``.occupancy`` surface of
``oracle.Fast`` (so ``gang_oracle.fast_place_gangs`` drives it unchanged) and the rules of include/islplace.h for a restricted range:

- the sub-inventory is the GPUs [lo, hi), node boundaries clipped to the range, every GPU keeping its node's table;
- FREE: gpu >= G, size 0 or start + size > 8 -> BAD_SPAN; a valid span on a GPU outside [lo, hi) -> FREED and not applied; inside ->
  applied.  Every FREE record echoes (gpu, start, size);
- ALLOC: placed -> the canonical GPU index; unplaced -> (GPU_NONE, 9, size) with the size of the WHOLE inventory's default
  (``gang_oracle.default_sizes``), not the sub-inventory's; unknown profile -> BAD_PROFILE;
- NOOP and every op value other than ALLOC / FREE -> NOOP;
- the bytes outside [lo, hi) never change.

``place_range`` is one call; with ``all_nodes=True`` it is ISL_FLAG_ALL_NODES: one restricted call per node of the clipped range in policy
order (right-to-left: last node first), each seeing the whole request array; a pod's record is that of the first pass that placed it, the
FREE records those of the first pass.

``capacity_by_hand`` is isl_capacity over a slice of the occupancy, repeating the start search byte by byte.
"""
from __future__ import annotations

import functools

import numpy as np

import oracle
from instaslice_b200 import engine as E
from instaslice_b200.workloads import alloc_requests

from gang_oracle import default_sizes


class RangeFast:
    def __init__(self, node_off, rows, occ, lo, hi, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None):
        self.node_off = np.asarray(node_off, dtype=np.int64)
        self.rows = np.asarray(rows)
        self.G = int(self.node_off[-1])
        assert 0 <= lo <= hi <= self.G
        self.lo, self.hi = int(lo), int(hi)
        self.occ = np.array(occ, dtype=np.uint8)
        assert len(self.occ) == self.G
        self.sizes = default_sizes(self.rows, node_table if node_table is not None else np.zeros(len(self.node_off) - 1, np.uint8))
        # the sub-inventory: node boundaries inside (lo, hi) plus the range's own ends; each clipped node keeps its node's table
        inner = [int(b) for b in self.node_off if self.lo < b < self.hi]
        sub_off = np.array([self.lo] + inner + [self.hi], dtype=np.int64) - self.lo
        sub_table = None
        if self.rows.ndim == 2:
            owner = np.searchsorted(self.node_off, sub_off[:-1] + self.lo, side="right") - 1
            sub_table = np.asarray(node_table, dtype=np.uint8)[np.minimum(owner, len(self.node_off) - 2)]
        self.sub = oracle.Fast(sub_off.astype(np.uint32), self.rows, quirks, policy, node_table=sub_table)
        self.sub.load(self.occ[self.lo:self.hi])

    def place(self, requests) -> np.ndarray:
        req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
        sub_req = req.copy()
        op = req["op"]
        g = req["handle"].astype(np.int64)
        start, size = req["start"].astype(np.int64), req["size"].astype(np.int64)
        free = op == E.OP_FREE
        bad = free & ((g >= self.G) | (size == 0) | (start + size > 8))     # ISL_SLOTS
        inside = free & ~bad & (g >= self.lo) & (g < self.hi)
        sub_req["handle"][inside] -= self.lo
        sub_req["op"][(free & ~inside) | ((op != E.OP_ALLOC) & ~free)] = E.OP_NOOP
        out = self.sub.place(sub_req)
        placed = (op == E.OP_ALLOC) & (out["status"] == E.ST_PLACED)
        out["gpu"][placed] += self.lo
        unplaced = np.flatnonzero((op == E.OP_ALLOC) & (out["status"] == E.ST_NO_CAPACITY))
        out["size"][unplaced] = [self.sizes[int(p)] for p in req["profile"][unplaced]]
        out["gpu"][free], out["start"][free], out["size"][free] = req["handle"][free], req["start"][free], req["size"][free]
        out["status"][free] = np.where(bad[free], E.ST_BAD_SPAN, E.ST_FREED)
        self.occ[self.lo:self.hi] = self.sub.occupancy()
        return out

    def occupancy(self) -> np.ndarray:
        return self.occ.copy()


OP_UNKNOWN = 7      # no op the engine knows: reported NOOP


def _busy_span(occ, g):
    """The first run of busy slices on GPU g (a live allocation), or slice 0 of an empty GPU."""
    b = int(occ[g])
    if b == 0:
        return 0, 1
    s = (b & -b).bit_length() - 1
    e = s
    while e < 8 and (b >> e) & 1:
        e += 1
    return s, e - s


def mixed_requests(rng, occ, lo, hi, n_names, n, profile=None):
    """ALLOCs (every profile, or ``profile`` alone) with, at random positions, at least one of each: a FREE of a busy span inside
    [lo, hi), a valid FREE of a busy span outside it, a malformed FREE (beyond G, size 0 or past slot 8), a NOOP, op 7 and an unknown
    profile; beyond 8 requests one in 16 is such a request."""
    G = len(occ)
    if profile is None:
        p = (rng.next(n) % np.uint64(n_names + 1)).astype(np.uint8)
        p[p == n_names] = E.PROFILE_UNKNOWN
    else:
        p = np.full(n, profile, dtype=np.uint8)
    req = alloc_requests(p)
    kinds = ["in", "out", "bad", "noop", "op7", "unknown"]
    slots = rng.next(n) % np.uint64(n)
    extra = [int(i) for i in np.flatnonzero(rng.next(n) % np.uint64(16) == 0)] if n > 8 else []
    todo = [(int(slots[k]), kinds[k]) for k in range(min(n, len(kinds)))] + [(i, kinds[i % len(kinds)]) for i in extra]
    for i, kind in todo:
        r = int(rng.next1())
        inside = hi > lo and (kind == "in" or lo == 0 and hi == G)
        if kind in ("in", "out"):
            if inside:
                g = lo + r % (hi - lo)
            else:
                outside = lo + (G - hi)
                if outside == 0:
                    continue
                g = r % outside
                g = g if g < lo else hi + (g - lo)
            s, z = _busy_span(occ, g)
            req[i] = (g, 0, E.OP_FREE, s, z)
        elif kind == "bad":
            req[i] = [(G + r % 3, 0, E.OP_FREE, 0, 1), (r % G, 0, E.OP_FREE, 3, 0), (r % G, 0, E.OP_FREE, 5, 4)][(r >> 8) % 3]
        elif kind == "noop":
            req["op"][i] = E.OP_NOOP
        elif kind == "op7":
            req["op"][i] = OP_UNKNOWN
        else:
            req["op"][i], req["profile"][i] = E.OP_ALLOC, E.PROFILE_UNKNOWN
    return req


def node_order(node_off, lo, hi, policy):
    """The clipped [a, b) of every node that meets [lo, hi), in the order ISL_FLAG_ALL_NODES visits them."""
    spans = [(max(lo, int(a)), min(hi, int(b))) for a, b in zip(node_off[:-1], node_off[1:])]
    spans = [(a, b) for a, b in spans if a < b]
    return spans[::-1] if policy == E.POLICY_RIGHT_TO_LEFT else spans


@functools.lru_cache(maxsize=None)
def _in_a_row(row_bytes, quirks):
    """[256]: for every occupancy byte, how many placements of the row the start search grants in a row."""
    row = np.frombuffer(row_bytes, dtype=E.PROFILE_DTYPE)[0]
    out = np.zeros(256, dtype=np.uint64)
    for o in range(256):
        b, k = o, 0
        while (s := oracle.start_for(row, quirks, b)) != E.START_NONE:
            b |= ((1 << int(row["size"])) - 1) << s
            k += 1
        out[o] = k
    return out


def capacity_by_hand(rows, quirks, occ, gpu_table=None):
    """cap[p] (MAX_PROFILES entries) over the occupancy bytes ``occ``: the placements of p alone that the start search grants in a row,
    summed over the GPUs.  ``rows``: [n_profiles], or [n_tables][n_profiles] with ``gpu_table`` the table of every GPU of ``occ``."""
    rows = np.asarray(rows, dtype=E.PROFILE_DTYPE)
    occ = np.asarray(occ, dtype=np.uint8)
    if rows.ndim == 1:
        rows, gpu_table = rows[None], np.zeros(len(occ), dtype=np.uint8)
    gpu_table = np.asarray(gpu_table, dtype=np.uint8)
    cap = np.zeros(E.MAX_PROFILES, dtype=np.uint64)
    for t in range(rows.shape[0]):
        counts = np.bincount(occ[gpu_table == t], minlength=256).astype(np.uint64)
        for p in range(rows.shape[1]):
            cap[p] += np.dot(_in_a_row(rows[t, p].tobytes(), quirks), counts)
    return cap


def place_range(node_off, rows, occ, lo, hi, requests, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
                all_nodes=False):
    """isl_place_batch_range(lo, hi, requests) on ``occ``: returns (records, the whole occupancy after the call)."""
    req = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    spans = node_order(node_off, lo, hi, policy) if all_nodes else [(lo, hi)]
    if not spans:
        spans = [(lo, lo)]          # an empty range: the defaults of one pass
    occ = np.array(occ, dtype=np.uint8)
    out = None
    for a, b in spans:
        ref = RangeFast(node_off, rows, occ, a, b, quirks, policy, node_table)
        res = ref.place(req)
        occ = ref.occupancy()
        if out is None:
            out = res
        else:
            take = (req["op"] == E.OP_ALLOC) & (out["status"] != E.ST_PLACED) & (res["status"] == E.ST_PLACED)
            out[take] = res[take]
    return out, occ
