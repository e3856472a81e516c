"""Profile alternatives (ISL_FLAG_FIRST_AVAILABLE, include/islplace.h A1-A8) at the limits of the ABI — the pod generators, their
self-checks and the pins of the checkers at these shapes (CPU only).  ``test_gpu_first_available_limits.py`` runs the same inputs through
k_bestfit<.., kAlt = true> (FIRST_FIT, BEST_FIT, RIGHT_TO_LEFT, MIN_FRAG) and k_nodefit<true> (MOST_ / LEAST_ALLOCATED).

The fixtures are those of ``test_oracle_table_limits.py`` and ``test_oracle_gang_topology_limits.py`` (T16x8, T16mix-1/2, T8tab with its
node tables, T16top, T16straddle); the occupancy and node shapes those of ``test_oracle_request_major_limits.py`` and the k_bestfit edges
those of ``test_oracle_bestfit_limits.py``.  Built here:
  podify         a request stream made pods of alternatives: runs of 1..6 ALLOCs, some profile bytes at or above the name count (15,
                 n_names, 16, 200, 254, 255), FREEs of single slices and of whole bytes, NOOPs and ops 3..255 between pods with equal
                 handles; 32-bit handles where neighbouring pods differ only in bit 16 or bit 31, and one pod with handle 0xFFFFFFFF
  edge_call      runs of 33, 64, 65 and 100 alternatives over two to four 32-request blocks (the placed one in the first block), pods
                 opening at lane 0 and at lane 31 behind an ALLOC, a NOOP and an op 3..255 of a handle equal in its low 16 bits
  dead15_call    T16top: profile 15 (size 8) has no empty GPU, dies as a pod's first alternative and stays dead for later pods of the block
                 and of later blocks; a second batch frees whole bytes and places profile 15 again
  wrap_pods      each ALLOC of a k_bestfit edge call (sparse_call, SWITCH_CASES, tie_call, only_top_call, top_call) made a pod: unknown
                 profile bytes in front, the same profile behind, so the pods take exactly the original call's GPUs
"""
import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

import bestfit_fast as BF
import first_available_fast as F
import first_available_oracle as O
from test_oracle_bestfit_limits import (HALF, SPARSE_G, SPARSE_LO, SWITCH_CASES, TOP, TOP_LO, Walk, frees_applied,
                                        lower_half_full, only_top_call, sparse_call, sparse_edges, span_of, switch_call, tie_call, top_call)
from test_oracle_gang_topology_limits import FIXTURES
from test_oracle_request_major_limits import eight_gpu_nodes, gang_call, gpu_tables, scoring_nodes, top_nodes, whole_bytes
from test_oracle_table_limits import candidate_mask, min_frag_scores, ragged_nodes, t16top, t16x8, t8tab, t8tab_node_tables

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG, E.POLICY_MOST_ALLOCATED,
            E.POLICY_LEAST_ALLOCATED]
BF_POLICIES = [E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG]
KBF_POLICIES = POLICIES[:4]                 # k_bestfit<.., kAlt>; the node-scoring two run k_nodefit<true>
NF_SMEM_NODES = 2048                        # kNfSmemNodes: up to here k_nodefit's score trees live in shared memory
ALL_STATUSES = {E.ST_PLACED, E.ST_NO_CAPACITY, E.ST_BAD_PROFILE, E.ST_ALT_SKIPPED, E.ST_FREED, E.ST_BAD_SPAN, E.ST_NOOP}
LONG_RUNS = (33, 64, 65, 100)
BIT16, BIT31 = 1 << 16, 1 << 31
# every fixture under every quirk set
ALL_CASES = [(f, q) for f in ("t16x8", "t16mix1", "t16mix2", "t8tab", "t16top", "t16straddle") for q in (0, 1, 2, 3)]


def odd_bytes(n_names):
    """Profile bytes at and above the name count (15 is a name of the 16-name fixtures)."""
    return (15, n_names, 16, 200, 254, 255)


def fa_place(*args, **kw):
    """The brute force with its score memo, which the 2^20-GPU ISL_POLICY_MIN_FRAG calls here need (``test_memo_on_equals_memo_off``
    pins it against the plain walk)."""
    return F.place(*args, memo=True, **kw)


def fixture_case(name, rng, G):
    """(rows, node_off, node_table) of a fixture on G GPUs of eight-GPU nodes, T8tab with its node tables."""
    rows = FIXTURES[name]()
    node_off = eight_gpu_nodes(G)
    return rows, node_off, t8tab_node_tables(rng, len(node_off) - 1) if rows.ndim == 2 else None


# ---- pod generators -----------------------------------------------------------------------------------------------------------------
class Handles:
    """Pod handles: each is the one before it with bit 16 or bit 31 flipped (they alternate), so neighbouring pods are equal in their low
    16 bits (and in their low 31 bits every other time); now and then a fresh random base, and once 0xFFFFFFFF."""

    def __init__(self, rng):
        self.rng, self.k = rng, 0
        self.h = int(rng.next1() & 0xFFFFFFFF)

    def next(self):
        self.k += 1
        if self.k == 7:
            self.h = 0xFFFFFFFF
        elif self.k % 23 == 0:
            self.h = int(self.rng.next1() & 0xFFFFFFFF)
        else:
            self.h ^= BIT16 if self.k % 2 else BIT31
        return self.h


def podify(rng, req, n_names, G, max_run=6):
    """A request stream (``gang_call``'s mix) made pods of alternatives.  Consecutive ALLOCs become pods of 1..max_run alternatives,
    about one in eight with a profile byte from ``odd_bytes``; a NOOP takes the handle of the pod before it, and so does the pod after it
    (two pods, A1), about half of them as an op 3..255 instead; about one FREE in three frees a whole byte and one in six reaches past
    slot 7 (BAD_SPAN)."""
    req = np.array(req, dtype=E.REQUEST_DTYPE)
    hs = Handles(rng)
    odd = odd_bytes(n_names)
    out, i, h, keep = [], 0, hs.h, False
    while i < len(req):
        r = req[i]
        if r["op"] == E.OP_ALLOC:
            k = 1 + int(rng.next1() % max_run)
            h = h if keep else hs.next()
            keep = False
            while k and i < len(req) and req[i]["op"] == E.OP_ALLOC:
                p = int(req[i]["profile"])
                if rng.next1() % 8 == 0:
                    p = odd[int(rng.next1() % len(odd))]
                out.append((h, p, E.OP_ALLOC, 0, 0))
                i, k = i + 1, k - 1
            continue
        if r["op"] == E.OP_FREE:
            kind = rng.next1() % 6
            if kind < 2:
                out.append((r["handle"], 0, E.OP_FREE, 0, 8))
            elif kind == 2:
                out.append((r["handle"], 0, E.OP_FREE, r["start"], 9 - int(r["start"])))
            else:
                out.append(tuple(r))
        else:
            op = E.OP_NOOP if rng.next1() % 2 else 3 + int(rng.next1() % 253)
            out.append((h, 0, op, 0, 0))
            keep = True
        i += 1
    return np.array(out, dtype=E.REQUEST_DTYPE)


def alt_call(rng, G, n_names, n, max_run=6):
    """``gang_call``'s mix of n requests made pods."""
    return podify(rng, gang_call(rng, G, n_names, n), n_names, G, max_run)


class Builder:
    """A call assembled at chosen positions of its 32-request blocks."""

    def __init__(self, rng, n_names):
        self.rng, self.n_names, self.req, self.hs = rng, n_names, [], Handles(rng)
        self.runs = []                      # (first request, length) of every long run
        self.marks = {}

    def pod(self, profiles, handle=None):
        """A pod; a chosen ``handle`` moves the chain to a fresh base, so that the next pod of one cannot take it too."""
        h = self.hs.next() if handle is None else handle
        if handle is not None:
            self.hs.h = int(self.rng.next1() & 0xFFFFFFFF)
        self.req.extend((h, int(p), E.OP_ALLOC, 0, 0) for p in profiles)
        return h

    def ones(self, k):
        for _ in range(k):
            self.pod([int(self.rng.next1() % self.n_names)])

    def pad_to(self, lane):
        self.ones((lane - len(self.req)) % 32)

    def run(self, length, good, lead=2):
        """A run of ``length`` alternatives: ``lead`` unknown profile bytes, the ``good`` ones, then known profiles (which would place if
        the pod were not done)."""
        head = [200, 255][:lead] + list(good)
        tail = [int(p) for p in self.rng.next(length - len(head)) % np.uint64(self.n_names)]
        self.runs.append((len(self.req), length))
        return self.pod(head + tail)

    def array(self):
        return np.array(self.req, dtype=E.REQUEST_DTYPE)


def edge_call(rng, n_names, good):
    """Long runs and block-edge openings; ``good``: profiles of which at least one places (the first, where a run opens at lane 31).
    Returns (requests, runs, marks); marks["lane30"]: the pod of five that opens at lane 30."""
    b = Builder(rng, n_names)
    b.ones(3)
    b.run(100, good)                                    # lanes 3..31 + 32 + 32 + 7: four blocks
    b.pad_to(0)
    b.run(33, good)                                     # opens at lane 0: 32 + 1
    b.pad_to(31)
    b.run(64, good[:1], lead=0)                         # opens at lane 31: 1 + 32 + 31
    b.pad_to(0)
    b.run(65, good)                                     # 32 + 32 + 1
    b.pad_to(31)
    h = b.pod([int(rng.next1() % n_names)])             # lane 31, then a pod at lane 0 whose handle differs from it in bit 16 only
    b.pod([int(rng.next1() % n_names)], h ^ BIT16)
    b.pad_to(31)
    h = b.pod([int(rng.next1() % n_names)])
    b.pod(list(good[:1]) * 3, h ^ BIT31)               # ... in bit 31 only
    b.pad_to(31)
    b.req.append((h, 0, 3 + int(rng.next1() % 253), 0, 0))      # lane 31: an op 3..255 carrying the handle of the pod at lane 0
    b.pod(list(good[:1]) * 2, h)
    b.pad_to(31)
    b.req.append((0xFFFFFFFF, 0, E.OP_NOOP, 0, 0))              # lane 31: a NOOP with the handle of the pod at lane 0
    b.pod([int(rng.next1() % n_names)] * 2, 0xFFFFFFFF)
    b.pad_to(30)
    b.marks["lane30"] = len(b.req)
    b.pod([good[0], good[0]], 0x7FFFFFFF)                       # lanes 30, 31 and on at lane 0 of the next block: one pod
    b.pod([good[0]] * 3, 0x7FFFFFFF)
    b.pad_to(31)
    b.run(64, good[:1], lead=0)
    b.ones(5)
    return b.array(), b.runs, b.marks


def good_profiles(rows, quirks):
    """Every name some table places in a row of its own, smallest first: at least one fits whole_bytes' empty GPUs."""
    rows2 = rows if rows.ndim == 2 else rows[None]
    out = []
    for p in range(rows2.shape[1]):
        sizes = [int(rows2[t, p]["size"]) for t in range(rows2.shape[0])
                 if any(candidate_mask(rows2[t, p]["size"], s, quirks) for s in rows2[t, p]["starts"][:rows2[t, p]["n_starts"]])]
        if sizes:
            out.append((min(sizes), p))
    return [p for _, p in sorted(out)][:3]


def wrap_pods(rng, req, n_names):
    """Each ALLOC of ``req`` made a pod: 0..2 unknown profile bytes, the ALLOC's profile, then 0..2 repeats of it (which fail where it
    failed and are skipped where it placed).  Every other request is kept.  The pods take exactly the GPUs the original call takes."""
    hs = Handles(rng)
    bad = [p for p in odd_bytes(n_names) if p >= n_names]
    out = []
    for r in req:
        if r["op"] != E.OP_ALLOC:
            out.append(tuple(r))
            continue
        h, p = hs.next(), int(r["profile"])
        alts = [bad[int(rng.next1() % len(bad))] for _ in range(int(rng.next1() % 3))] + [p] * (1 + int(rng.next1() % 3))
        out.extend((h, a, E.OP_ALLOC, 0, 0) for a in alts)
    return np.array(out, dtype=E.REQUEST_DTYPE)


def every_status_tail(occ, G, lo, hi):
    """Requests that leave the occupancy as it is and add the records an edge call lacks: a FREE of a slice that is already free
    (FREED), FREEs past the inventory and past slot 7 (BAD_SPAN), a NOOP, an op 3..255 and a pod of unknown profile bytes."""
    g = lo + int(np.flatnonzero(occ[lo:hi] != 0xFF)[0])
    s = int(np.flatnonzero([not (int(occ[g]) >> k) & 1 for k in range(8)])[0])
    return np.array([(g, 0, E.OP_FREE, s, 1), (G, 0, E.OP_FREE, 0, 1), (g, 0, E.OP_FREE, 7, 2), (5, 0, E.OP_NOOP, 0, 0),
                     (5, 0, 200, 0, 0), (9, 254, E.OP_ALLOC, 0, 0), (9, 255, E.OP_ALLOC, 0, 0)], dtype=E.REQUEST_DTYPE)


def edge_pods(rng, kind, policy=E.POLICY_BEST_FIT, where="whole"):
    """A k_bestfit edge call as pods: (rows, quirks, node_off, node_table, occ, requests, lo, hi).  ``kind``: "sparse" (``where``:
    "whole" = SPARSE_G GPUs, "partition" = [777, 2^20)), "tie", "only_top", "t16top", "t16straddle" or a SWITCH_CASES name."""
    node_table, lo, hi = None, 0, None
    if kind == "sparse":
        G, lo, hi = (SPARSE_G, 0, SPARSE_G) if where == "whole" else (TOP, SPARSE_LO, TOP)
        rows, quirks, node_off, occ, req, _off = sparse_call(G, lo, hi, policy)
    elif kind == "tie":
        rows, quirks, node_off, occ, req = tie_call()
    elif kind == "only_top":
        rows, quirks, node_off, occ, req = only_top_call()
    elif kind in ("t16top", "t16straddle"):
        rows, quirks, node_off, occ, req = top_call(rng, kind, n=120)
    else:
        case = next(c for c in SWITCH_CASES if c[0] == kind)
        rows, quirks, node_off, node_table, occ, req, lo, hi = switch_call(rng, case, 300)
    G = int(node_off[-1])
    hi = G if hi is None else hi
    n_names = rows.shape[-1]
    req = np.concatenate([wrap_pods(rng, req, n_names), every_status_tail(occ, G, lo, hi)])
    return rows, quirks, node_off, node_table, occ, req, lo, hi


EDGE_KINDS = ["tie", "only_top", "t16top", "t16straddle"] + [c[0] for c in SWITCH_CASES]


def dead15_call(rng, G=4096, k=5):
    """T16top, FIXED quirks, eight-GPU nodes: no GPU empty (so profile 15, the size-8 row, fits nowhere), k of them full.  Batch 1: the
    pod [15, a] at lane 0 (15 dies, a places), [15, 15, b] at lane 9, [15, c] at lane 31 of block 2 and on, pods of one between.  Batch 2:
    whole-byte FREEs of the k full GPUs, then k + 1 pods [15, d]: 15 places k times and dies again.  Returns (rows, quirks, node_off,
    occ, batch 1, batch 2, the full GPUs)."""
    rows = t16top()
    node_off = eight_gpu_nodes(G)
    occ = whole_bytes(rng, G)
    occ[occ == 0] = 0x10
    full = np.flatnonzero(occ == 0xFF)[:k]
    assert len(full) == k
    b = Builder(rng, 15)
    b.pod([15, int(rng.next1() % 15)])
    b.ones(7)
    b.pod([15, 15, int(rng.next1() % 15)])
    b.pad_to(0)
    b.ones(32 + 31)
    b.pod([15, int(rng.next1() % 15)])
    b.ones(4)
    batch1 = b.array()
    frees = np.array([(int(g), 0, E.OP_FREE, 0, 8) for g in full], dtype=E.REQUEST_DTYPE)
    b2 = Builder(rng, 15)
    for _ in range(k + 1):
        b2.pod([15, int(rng.next1() % 15)])
    return rows, E.QUIRKS_FIXED, node_off, occ, batch1, np.concatenate([frees, b2.array()]), full


def top_range(rng, G=TOP, n=150):
    """T8tab on 2^20 GPUs of eight-GPU nodes, the lower half full (``lower_half_full``) and so every GPU of table 7, the only one that
    knows profile 15; pods of its mix, and the range from the first GPU past the first node on table 7 to the top: (rows, node_off,
    node_table, occ, requests, lo, hi)."""
    rows, node_off, node_table, occ, req = lower_half_full(rng, G, n)
    occ[gpu_tables(node_off, node_table) == 7] = 0xFF
    v7 = int(np.flatnonzero(node_table == 7)[0])
    lo = int(node_off[v7 + 1]) + 3
    return rows, node_off, node_table, occ, np.concatenate([podify(rng, req, 16, G), every_status_tail(occ, G, lo, G)]), lo, G


def admits_table(rows, quirks):
    """[table][profile][byte]: the profile has a legal free start on a GPU of that table with that byte."""
    rows2 = rows if rows.ndim == 2 else rows[None]
    out = np.zeros(rows2.shape[:2] + (256,), dtype=bool)
    for t, p in np.ndindex(rows2.shape[:2]):
        r = rows2[t, p]
        masks = [m for m in (candidate_mask(r["size"], s, quirks) for s in r["starts"][:r["n_starts"]]) if m]
        for o in range(256):
            out[t, p, o] = any(not o & m for m in masks)
    return out


def pods_of(req):
    """[(first, end)] of every pod (A1)."""
    opens = np.flatnonzero(O.pod_starts(req))
    out = []
    for a in opens:
        b = a + 1
        while b < len(req) and req["op"][b] == E.OP_ALLOC and req["handle"][b] == req["handle"][a]:
            b += 1
        out.append((int(a), int(b)))
    return out


def check_a5a(rows, quirks, node_off, node_table, occ, req, out, lo, hi):
    """A5 (a): replaying the records, each pod's PLACED alternative is the first one some GPU of [lo, hi) admits at that moment, and a
    pod without one has no admitting GPU for any of its known alternatives."""
    adm = admits_table(rows, quirks)
    nt = np.zeros(len(node_off) - 1, np.uint8) if node_table is None else node_table
    gtab = gpu_tables(node_off, nt)[lo:hi].astype(np.int64)
    live = frees_applied(occ, req, lo, hi)
    n_names = adm.shape[1]
    for a, b in pods_of(req):
        st = out["status"][a:b]
        placed = np.flatnonzero(st == E.ST_PLACED)
        k = int(placed[0]) if len(placed) else b - a
        assert (st[k + 1:] == E.ST_ALT_SKIPPED).all()
        for i in range(a, a + k):
            p = int(req["profile"][i])
            assert st[i - a] == (E.ST_NO_CAPACITY if p < n_names else E.ST_BAD_PROFILE)
            if p < n_names:
                assert not adm[gtab, p, live[lo:hi]].any(), (i, p)
        if len(placed):
            i = a + k
            g, span = int(out["gpu"][i]), span_of(out[i])
            assert lo <= g < hi and adm[gtab[g - lo], int(req["profile"][i]), live[g]] and not int(live[g]) & span
            live[g] |= span


def walk_of(node_off, node_table, occ, req, out, lo, hi, policy):
    """The records' placements replayed on a ``Walk`` of k_bestfit's classes."""
    nt = np.zeros(len(node_off) - 1, np.uint8) if node_table is None else node_table
    walk = Walk(frees_applied(occ, req, lo, hi), gpu_tables(node_off, nt), lo, hi, policy == E.POLICY_RIGHT_TO_LEFT)
    for r in out[out["status"] == E.ST_PLACED]:
        walk.take(int(r["gpu"]), span_of(r))
    return walk


def statuses(*outs):
    return set(int(s) for o in outs for s in np.unique(o["status"]))


# ---- the checkers agree ------------------------------------------------------------------------------------------------------------
def _same(a, b, what):
    bad = np.flatnonzero(a[0] != b[0])
    assert len(bad) == 0, (what, bad[:4], a[0][bad[:4]], b[0][bad[:4]])
    assert np.array_equal(a[1], b[1]) and a[2] == b[2], what


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", ALL_CASES, ids=["%s-q%d" % c for c in ALL_CASES])
def test_brute_force_equals_the_composition(name, quirks, policy):
    """first_available_fast against first_available_oracle on ragged inventories with empty nodes: the whole inventory, a range and a
    partition that cut nodes at both ends, and the block-edge call."""
    rows = FIXTURES[name]()
    n_names = rows.shape[-1]
    rng = W.SplitMix64(7000 + 100 * policy + 10 * quirks + len(name))
    seen = set()
    for trial in range(3):
        node_off = scoring_nodes(rng, 24 + int(rng.next1() % 24))
        G = int(node_off[-1])
        node_table = t8tab_node_tables(rng, len(node_off) - 1) if rows.ndim == 2 else None
        occ = whole_bytes(rng, G)
        req = alt_call(rng, G, n_names, 160)
        cut = [v for v in range(1, len(node_off) - 1) if node_off[v + 1] - node_off[v] >= 3]
        lo, hi = (0, G) if trial == 0 else (int(node_off[cut[trial - 1]]) + 1, int(node_off[cut[-trial] + 1]) - 1)
        a = fa_place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
        _same(a, O.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi), (trial, lo, hi))
        seen |= statuses(a[0])
    node_off = scoring_nodes(rng, 60)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1) if rows.ndim == 2 else None
    occ = whole_bytes(rng, G)
    req = edge_call(rng, n_names, good_profiles(rows, quirks) or [0])[0]
    _same(fa_place(node_off, rows, occ, req, policy, quirks, node_table), O.place(node_off, rows, occ, req, policy, quirks, node_table),
          "edge call")
    assert {E.ST_PLACED, E.ST_BAD_PROFILE, E.ST_ALT_SKIPPED, E.ST_FREED, E.ST_BAD_SPAN, E.ST_NOOP} <= seen


@pytest.mark.parametrize("policy", POLICIES)
def test_dead15_call_against_the_composition(policy):
    rng = W.SplitMix64(1515 + policy)
    rows, quirks, node_off, occ, b1, b2, _full = dead15_call(rng, G=512, k=3)
    a1 = fa_place(node_off, rows, occ, b1, policy, quirks)
    _same(a1, O.place(node_off, rows, occ, b1, policy, quirks), "batch 1")
    _same(fa_place(node_off, rows, a1[1], b2, policy, quirks), O.place(node_off, rows, a1[1], b2, policy, quirks), "batch 2")


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name", ["t8tab", "t16top", "t16straddle", "t16x8"])
def test_memo_on_equals_memo_off(name, policy):
    rows = FIXTURES[name]()
    quirks = E.QUIRKS_REF_EXACT if name == "t16x8" else E.QUIRKS_FIXED
    rng = W.SplitMix64(4200 + policy + len(name))
    for G in (64, 777):
        rows_, node_off, node_table = fixture_case(name, rng, G)
        occ = whole_bytes(rng, G)
        req = alt_call(rng, G, rows.shape[-1], 300)
        a = F.place(node_off, rows, occ, req, policy, quirks, node_table, 3, G - 2, memo=True)
        b = F.place(node_off, rows, occ, req, policy, quirks, node_table, 3, G - 2, memo=False)
        _same(a, b, G)
        assert a[2] > 0


# ---- the generators reach their edges ------------------------------------------------------------------------------------------------
def test_podify_reaches_every_request_edge():
    rng = W.SplitMix64(16)
    G = 4096
    req = alt_call(rng, G, 16, 3000)
    pods = pods_of(req)
    lengths = {b - a for a, b in pods}
    assert set(range(1, 7)) <= lengths
    prof = req["profile"][req["op"] == E.OP_ALLOC]
    assert set(odd_bytes(16)) <= set(prof.tolist())
    ops = req["op"].tolist()
    assert E.OP_NOOP in ops and any(3 <= o <= 255 for o in ops)
    frees = req[req["op"] == E.OP_FREE]
    assert ((frees["size"] == 8) & (frees["start"] == 0)).any() and (frees["size"] == 1).any()
    assert (frees["start"].astype(int) + frees["size"] > 8).any()
    # between pods of equal handles: a NOOP and an op 3..255
    split = [i for i in range(1, len(req) - 1) if req["op"][i] not in (E.OP_ALLOC, E.OP_FREE) and req["op"][i - 1] == E.OP_ALLOC
             and req["op"][i + 1] == E.OP_ALLOC and req["handle"][i - 1] == req["handle"][i + 1]]
    assert {req["op"][i] == E.OP_NOOP for i in split} == {True, False}
    # neighbouring pods differ in bit 16 only and in bit 31 only; one pod is 0xFFFFFFFF
    h = [int(req["handle"][a]) for a, _ in pods]
    diffs = {a ^ b for a, b in zip(h, h[1:])}
    assert BIT16 in diffs and BIT31 in diffs and 0xFFFFFFFF in h
    adjacent = [i for i in range(1, len(req)) if req["op"][i] == req["op"][i - 1] == E.OP_ALLOC
                and req["handle"][i] != req["handle"][i - 1]]
    assert {int(req["handle"][i] ^ req["handle"][i - 1]) for i in adjacent} >= {BIT16, BIT31}


@pytest.mark.parametrize("name,quirks", [("t16x8", E.QUIRKS_REF_EXACT), ("t8tab", E.QUIRKS_FIXED), ("t16mix2", 1), ("t16mix1", 2)])
def test_edge_call_carries_pods_across_block_edges(name, quirks):
    """Every long run places in its first block and skips every alternative in two or three later blocks; pods open at lane 0 behind an
    ALLOC, a NOOP and an op 3..255 whose handles equal the pod's in their low 16 bits, and one pod runs from lane 30 across the edge."""
    rng = W.SplitMix64(33 + quirks)
    rows, node_off, node_table = fixture_case(name, rng, 4096)
    occ = whole_bytes(rng, 4096)
    good = good_profiles(rows, quirks)
    req, runs, marks = edge_call(rng, rows.shape[-1], good)
    assert sorted(n for _, n in runs) == sorted(LONG_RUNS + (64,))
    for policy in POLICIES:
        out, _, _ = fa_place(node_off, rows, occ, req, policy, quirks, node_table)
        blocks = set()
        for a, n in runs:
            st = out["status"][a:a + n]
            k = int(np.flatnonzero(st == E.ST_PLACED)[0])
            assert (a + k) // 32 == a // 32 and (st[k + 1:] == E.ST_ALT_SKIPPED).all(), (policy, a, n)
            blocks.add((a + n - 1) // 32 - a // 32)
        assert blocks == {1, 2, 3}
        # the pods opening at lane 0
        lane0 = [i for i in range(32, len(req), 32) if req["op"][i] == E.OP_ALLOC and O.pod_starts(req)[i]]
        before = {(int(req["op"][i - 1]) if req["op"][i - 1] != E.OP_ALLOC else -1) for i in lane0
                  if int(req["handle"][i - 1]) & 0xFFFF == int(req["handle"][i]) & 0xFFFF}
        assert -1 in before and E.OP_NOOP in before and any(3 <= o <= 255 for o in before)
        i = marks["lane30"]
        assert i % 32 == 30 and req["handle"][i] == 0x7FFFFFFF
        assert not O.pod_starts(req)[i + 1:i + 5].any() and out["status"][i] == E.ST_PLACED
        assert (out["status"][i + 1:i + 5] == E.ST_ALT_SKIPPED).all()


@pytest.mark.parametrize("policy", POLICIES)
def test_profile_15_dies_within_a_launch_only(policy):
    rng = W.SplitMix64(4096 + policy)
    rows, quirks, node_off, occ, b1, b2, full = dead15_call(rng)
    out1, occ1, _ = fa_place(node_off, rows, occ, b1, policy, quirks)
    pods = pods_of(b1)
    fifteen = [(a, b) for a, b in pods if b1["profile"][a] == 15]
    assert [a % 32 for a, _ in fifteen] == [0, 9, 31] and [a // 32 for a, _ in fifteen] == [0, 0, 2]
    for a, b in fifteen:
        st = out1["status"][a:b].tolist()
        assert st == [E.ST_NO_CAPACITY] * (b - a - 1) + [E.ST_PLACED], (a, st)
        assert out1["size"][a] == 8
    assert not (occ1 == 0).any()
    out2, occ2, _ = fa_place(node_off, rows, occ1, b2, policy, quirks)
    allocs = out2[b2["op"] == E.OP_ALLOC].reshape(-1, 2)
    k = len(full)
    assert (allocs[:k, 0]["status"] == E.ST_PLACED).all() and (allocs[:k, 1]["status"] == E.ST_ALT_SKIPPED).all()
    assert sorted(allocs[:k, 0]["gpu"].tolist()) == sorted(full.tolist())
    assert allocs[k, 0]["status"] == E.ST_NO_CAPACITY and allocs[k, 1]["status"] == E.ST_PLACED


@pytest.mark.parametrize("policy", KBF_POLICIES)
@pytest.mark.parametrize("where", ["whole", "partition"])
def test_sparse_pods_reach_every_branch_of_the_walk(where, policy):
    """The pods of sparse_call take its GPUs, and their placements replayed on the Walk reach every branch of min_after."""
    rng = W.SplitMix64(777 + policy)
    rows, quirks, node_off, node_table, occ, req, lo, hi = edge_pods(rng, "sparse", policy, where)
    out, _after, placed = fa_place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
    _r, _q, _n, occ0, req0, _off = sparse_call(int(node_off[-1]), lo, hi, policy)
    want, _ = BF.place(node_off, rows, occ0, req0, quirks, policy, lo=lo, hi=hi)
    assert out["gpu"][out["status"] == E.ST_PLACED].tolist() == want["gpu"][want["status"] == E.ST_PLACED].tolist() and placed == 7
    walk = walk_of(node_off, node_table, occ, req, out, lo, hi, policy)
    assert all(sparse_edges(walk, hi - lo).values()), sparse_edges(walk, hi - lo)
    assert statuses(out) == ALL_STATUSES
    if policy in BF_POLICIES:
        check_a5a(rows, quirks, node_off, node_table, occ, req, out, lo, hi)


@pytest.mark.parametrize("kind", EDGE_KINDS)
def test_edge_pods_take_the_edge_calls_gpus(kind):
    """tie_call, only_top_call, top_call and the SWITCH_CASES as pods place exactly where the calls themselves do, under best-fit and
    min-frag; T16top / T16straddle reach min-frag scores above 63, the tie call places on both sides of 2^19."""
    for policy in BF_POLICIES:
        rng = W.SplitMix64(2020 + len(kind))
        rows, quirks, node_off, node_table, occ, req, lo, hi = edge_pods(rng, kind, policy)
        out, _, _ = fa_place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
        plain = req[(req["op"] == E.OP_ALLOC) & (req["profile"] < rows.shape[-1])]
        first = np.concatenate([[True], plain["handle"][1:] != plain["handle"][:-1]])
        unwrapped = plain[first].copy()
        want, _ = BF.place(node_off, rows, frees_applied(occ, req, lo, hi), unwrapped, quirks, policy, node_table, lo, hi)
        assert out["gpu"][out["status"] == E.ST_PLACED].tolist() == want["gpu"][want["status"] == E.ST_PLACED].tolist()
        assert statuses(out) >= ALL_STATUSES - {E.ST_NO_CAPACITY}          # the tie and one-GPU calls run out of room as well
        assert (E.ST_NO_CAPACITY in statuses(out)) >= (kind in ("tie", "only_top"))
        gpus = out["gpu"][out["status"] == E.ST_PLACED]
        if kind == "tie":
            assert (gpus == HALF - 1).any() and (gpus >= HALF).any()
        if kind == "only_top":
            assert gpus.tolist() == [TOP - 1]
        if kind in ("t16top", "t16straddle"):          # profile 15 places, with min-frag scores above 63 (and below 64) in play
            seen = min_frag_scores(rows, quirks)[15][occ]
            assert ((req["profile"] == 15) & (out["status"] == E.ST_PLACED)).any() and seen.max() > 63
            assert (kind == "t16top") or 0 < seen[seen > 0].min() < 64


@pytest.mark.parametrize("policy", POLICIES)
def test_top_range_places_above_bit_19_with_the_default_size_of_table_7(policy):
    """2^20 GPUs, T8tab: placements at GPU indices with bit 19 set; on the range that starts past the first node of table 7, the
    NO_CAPACITY and ALT_SKIPPED records of profile 15 carry table 7's size (the inventory's default), not 0."""
    rng = W.SplitMix64(TOP + policy)
    rows, node_off, node_table, occ, req, lo, hi = top_range(rng, n=120 if policy in (E.POLICY_MOST_ALLOCATED,
                                                                                    E.POLICY_LEAST_ALLOCATED) else 150)
    for a, b in ((0, TOP), (lo, hi)):
        out, _, _ = fa_place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table, a, b)
        placed = out[out["status"] == E.ST_PLACED]
        assert (placed["gpu"] >= HALF).any() and ((placed["gpu"] & HALF) != 0).any()
        assert statuses(out) == ALL_STATUSES
    v7 = int(np.flatnonzero(node_table == 7)[0])
    assert lo > int(node_off[v7])
    p15 = (req["op"] == E.OP_ALLOC) & (req["profile"] == 15)
    st = out["status"][p15]
    assert (st == E.ST_NO_CAPACITY).any() or (st == E.ST_ALT_SKIPPED).any()
    assert (out["size"][p15 & (out["status"] != E.ST_PLACED)] == rows["size"][7, 15]).all()


def test_default_size_on_a_range_without_table_7():
    """A range with no node of table 7: profile 15 fits nowhere in it, yet its records carry table 7's size."""
    rows = t8tab()
    rng = W.SplitMix64(715)
    node_off = ragged_nodes(rng, 60)
    node_table = t8tab_node_tables(rng, 60)
    node_table[node_table == 7] = 3
    node_table[40] = 7
    occ = whole_bytes(rng, int(node_off[-1]))
    lo, hi = int(node_off[0]) + 1, int(node_off[40])
    b = Builder(rng, 16)
    for _ in range(20):
        b.pod([15, 15, int(rng.next1() % 15), 15])
    req = b.array()
    for policy in POLICIES:
        out, _, _ = fa_place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table, lo, hi)
        p15 = req["profile"] == 15
        assert (out["status"][p15] != E.ST_PLACED).all() and (out["status"][p15] == E.ST_ALT_SKIPPED).any()
        assert (out["size"][p15] == rows["size"][7, 15]).all() and rows["size"][7, 15] != 0


@pytest.mark.parametrize("extra", [0, 1])
def test_scoring_node_counts_sit_on_both_sides_of_the_tree_switch(extra):
    rng = W.SplitMix64(2048 + extra)
    node_off = scoring_nodes(rng, NF_SMEM_NODES + extra)
    assert (len(node_off) - 1 <= NF_SMEM_NODES) == (extra == 0) and (np.diff(node_off.astype(np.int64)) == 0).any()
    top = top_nodes(W.SplitMix64(20))
    assert len(top) - 1 == 1 << 20 and int(top[-1]) <= TOP and (np.diff(top.astype(np.int64)) == 0).any()


@pytest.mark.parametrize("policy", POLICIES)
def test_a5a_at_the_limits(policy):
    """A5 (a) on the brute force: the 2^20-GPU T8tab call, the block-edge call on T16x8 and on T8tab with 8 tables of ragged nodes."""
    rng = W.SplitMix64(5000 + policy)
    rows, node_off, node_table, occ, req, lo, hi = top_range(rng, n=80)
    out, _, _ = fa_place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table, lo, hi)
    check_a5a(rows, E.QUIRKS_FIXED, node_off, node_table, occ, req, out, lo, hi)
    for name, quirks in (("t16x8", E.QUIRKS_REF_EXACT), ("t8tab", E.QUIRKS_FIXED)):
        rows = FIXTURES[name]()
        node_off = scoring_nodes(rng, 300)
        G = int(node_off[-1])
        node_table = t8tab_node_tables(rng, len(node_off) - 1) if rows.ndim == 2 else None
        occ = whole_bytes(rng, G, dense=True)
        req = np.concatenate([edge_call(rng, rows.shape[-1], good_profiles(rows, quirks))[0], alt_call(rng, G, rows.shape[-1], 400)])
        lo, hi = int(node_off[5]) + 1, G - 3
        out, _, _ = fa_place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
        check_a5a(rows, quirks, node_off, node_table, occ, req, out, lo, hi)
