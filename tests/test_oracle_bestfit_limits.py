"""k_bestfit at the inventory limits — the checker ``bestfit_fast``, a restatement of the kernel's class-minimum walk, the generators that
reach each edge of that walk and their self-checks (CPU only).  ``test_gpu_bestfit_limits.py`` runs the same inputs through the kernel.

k_bestfit keeps, per class (node table, occupancy byte), a two-level bitmap over the GPUs of the range (32 GPUs per word, 1 024 per
summary word) and the class minimum.  When a placement takes the minimum, ``min_after`` finds the next member: the summary word that held
the old minimum, else windows of 32 summary words (32 768 GPUs) from the next one, the lanes past W1 (the summary word count) reading 0.
``Walk`` restates that structure over the range in storage order (right-to-left stores the inventory reversed) and replays a call from
the checker's records, so each generator can show which branch of the walk it reaches:

  sparse_call     background bytes no profile of the call admits and a few beacons: the next member found in the second window and in
                  a later one, in the last, partial window of a range with Gr % 1 024 != 0, a class that empties after walking every
                  window to W1 (kInf), and an emptied class filled again by a later placement
  abort_call      a gang takes three beacons a window or more apart and fails: the abort puts them back, the minimum of the class they
                  left is restored and that of the class they entered is walked again over 28 windows; the next gang takes them back
  live_call       8 tables x 256 bytes: all 2 048 classes populated (64 per lane)
  switch_cases    one table at Gr = 4 096 (class bitmaps in shared memory) and 4 097 (global memory), whole and as unaligned partitions
                  of 2^20 GPUs, and 8 tables at Gr = 4 096 (global memory)
  tie_call        best-fit and min-frag ties between a GPU below 2^19 and GPUs at or above it; only_top_call: GPU 2^20 - 1 alone admits
                  the profile; top_call: T16top / T16straddle min-frag scores above 63 in the key's top byte
"""
import time

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

import bestfit_fast as BF
import gang_oracle as GO
import range_oracle as RO
from test_oracle_gang_topology_limits import CASES, FIXTURES, case_ids, cluster, small_gangs
from test_oracle_request_major_limits import GANG_SHAPES, eight_gpu_nodes, gang_call, gang_offsets, gang_sizes, whole_bytes
from test_oracle_table_limits import min_frag_scores, t16mix, t16x8, t8tab

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
BF_POLICIES = [E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG]
INF = 0xFFFFFFFF
BF_SMEM_GPUS = 4096                 # kBfSmemGpus: up to here the class bitmaps of one table live in shared memory
TOP = 1 << 20                       # kBfMaxGpus
SPARSE_G = TOP - 613                # a whole inventory with Gr % 1 024 == 411
SPARSE_LO = 777                     # a partition [777, 2^20): Gr % 1 024 == 247
TOP_LO = TOP - 4109                 # the top partition of the right-to-left gangs


# ---- k_bestfit's class structure, restated ---------------------------------------------------------------------------------------------
def bitmaps_in_smem(n_tables, Gr):
    """prepare_bestfit / k_bestfit: the class bitmaps live in shared memory for one table up to kBfSmemGpus GPUs, else in global."""
    return n_tables == 1 and Gr <= BF_SMEM_GPUS


class Walk:
    """The classes of the range [lo, hi) in storage order, replayed from a call's records.  ``edges`` collects what ``min_after`` did:
    ("word",) the next member under the old minimum's summary word; ("window", w, partial, last_word) found in window w (0: the first) of
    32 summary words, partial when the window reaches past W1, last_word when the member is in summary word W1 - 1; ("inf", windows) the
    class is empty after walking that many windows; ("refill",) a class that had become empty gets a member; ("abort_min",) an aborted
    member was the minimum of the class it had entered; ("restore", distance) an aborted member is again the minimum of its old class,
    ``distance`` summary words below the minimum it replaces."""

    def __init__(self, occ, gtab, lo, hi, flip):
        self.lo, self.hi, self.flip = lo, hi, flip
        self.Gr = hi - lo
        self.W1 = ((self.Gr + 31) // 32 + 31) // 32
        self.cls = self.local(gtab.astype(np.int64)) * 256 + self.local(occ)
        self.s_min = {}
        for c in np.unique(self.cls):
            self.s_min[int(c)] = int(np.flatnonzero(self.cls == c)[0])
        self.edges = []
        self.empty = set()

    def local(self, a):
        a = np.asarray(a)[self.lo:self.hi]
        return a[::-1].astype(np.int64) if self.flip else a.astype(np.int64)

    def pos(self, gpu):
        return self.hi - 1 - gpu if self.flip else gpu - self.lo

    def min_after(self, c, g):
        """min_after(class c, g): g has left c and no member of c lies below it."""
        m = np.flatnonzero(self.cls == c)
        assert len(m) == 0 or m[0] > g
        k = g >> 10
        if len(m) and m[0] >> 10 == k:                 # the summary word that held g
            self.edges.append(("word",))
            return int(m[0])
        k0, w = k + 1, 0
        while k0 < self.W1:                             # windows of 32 summary words; lane l reads word k0 + l if k0 + l < W1
            words = m >> 10
            hit = m[(words >= k0) & (words < min(k0 + 32, self.W1))]
            if len(hit):
                self.edges.append(("window", w, k0 + 32 > self.W1, int(hit[0]) >> 10 == self.W1 - 1))
                return int(hit[0])
            k0, w = k0 + 32, w + 1
        self.edges.append(("inf", w))
        return INF

    def enter(self, c, g):
        if self.s_min.get(c, INF) == INF and c in self.empty:
            self.edges.append(("refill",))
        self.s_min[c] = min(self.s_min.get(c, INF), g)

    def take(self, gpu, span):
        """A placement of ``span`` on canonical ``gpu``: it must be its class minimum (the kernel's key carries only that)."""
        g = self.pos(gpu)
        c0 = int(self.cls[g])
        assert self.s_min[c0] == g, (gpu, c0, self.s_min[c0])
        c1 = c0 | span
        self.cls[g] = c1
        self.enter(c1, g)
        self.s_min[c0] = self.min_after(c0, g)
        if self.s_min[c0] == INF:
            self.empty.add(c0)

    def give_back(self, gpu, span):
        """abort_gang: the member on canonical ``gpu`` leaves class c2 for c2 & ~span."""
        g = self.pos(gpu)
        c2 = int(self.cls[g])
        c = c2 & ~span
        was_min = self.s_min[c2] == g
        self.cls[g] = c
        old = self.s_min.get(c, INF)
        if g < old:
            self.edges.append(("restore", INF if old == INF else (old >> 10) - (g >> 10)))
        self.enter(c, g)
        if was_min:
            self.edges.append(("abort_min",))
            self.s_min[c2] = self.min_after(c2, g)


def span_of(rec):
    return ((1 << int(rec["size"])) - 1) << int(rec["start"])


def frees_applied(occ, req, lo, hi):
    occ = np.array(occ, dtype=np.uint8)
    for r in req[req["op"] == E.OP_FREE]:
        g, s, z = int(r["handle"]), int(r["start"]), int(r["size"])
        if lo <= g < hi and z and s + z <= 8:
            occ[g] &= ~(((1 << z) - 1) << s) & 0xFF
    return occ


def replay(node_off, rows, occ, req, gang_off, quirks, policy, node_table=None, lo=0, hi=None):
    """Run the checker on the call, then replay it on a ``Walk``: committed gangs member by member, an aborted gang's tentative
    placements (the checker on its members before the failure) and their undoing in reverse.  Returns (records, occupancy, walk)."""
    G = len(occ)
    hi = G if hi is None else hi
    out, after = BF.place_gangs(node_off, rows, occ, req, gang_off, quirks, policy, node_table, lo, hi)
    nt = np.zeros(len(node_off) - 1, np.uint8) if node_table is None else np.asarray(node_table, np.uint8)
    gtab = np.repeat(nt, np.diff(np.asarray(node_off, dtype=np.int64)))
    cur = frees_applied(occ, req, lo, hi)
    walk = Walk(cur, gtab, lo, hi, policy == E.POLICY_RIGHT_TO_LEFT)
    for a, b in zip(gang_off[:-1], gang_off[1:]):
        idx = [i for i in range(int(a), int(b)) if req["op"][i] == E.OP_ALLOC]
        st = out["status"][idx]
        if len(idx) and (st == E.ST_PLACED).all():
            for i in idx:
                walk.take(int(out["gpu"][i]), span_of(out[i]))
                cur[int(out["gpu"][i])] |= span_of(out[i])
            continue
        failed = [i for i in idx if out["status"][i] != E.ST_GANG_ABORTED]
        before = [i for i in idx if i < failed[0]] if failed else []
        if not before:
            continue
        sub = req[before].copy()
        tent, _ = BF.place(node_off, rows, cur, sub, quirks, policy, node_table, lo, hi)
        assert (tent["status"] == E.ST_PLACED).all()
        for r in tent:
            walk.take(int(r["gpu"]), span_of(r))
        for r in tent[::-1]:
            walk.give_back(int(r["gpu"]), span_of(r))
    return out, after, walk


# ---- generators ------------------------------------------------------------------------------------------------------------------------
Y_BYTE, Z_BYTE, X_BYTE = 0xFD, 0x7F, 0xFC     # T16x8 profile 0: slot 1 / slot 7 / slots 0 and 1 free; background 0xFF


def place_at(occ, lo, hi, flip, x, byte):
    """Occupancy byte of the GPU at storage-local position x of [lo, hi)."""
    occ[hi - 1 - x if flip else lo + x] = byte


def sparse_call(G, lo, hi, policy, gangs=False):
    """T16x8, REF_EXACT quirks, background 0xFF.  Storage-local beacons: Y (one free slot) at 5, 40 K + 17, (W1 - 10) K + 100 and
    Gr - 3; Z (one free slot) at 9; X (two free slots) at Gr - 1.  Nine ALLOCs of profile 0 take, under every policy, 5 (the next Y is
    found in window 1), 9 (Z empties after every window), 40 K + 17 (next Y in a later window), (W1 - 10) K + 100 (next Y in the last,
    partial window, in summary word W1 - 1), Gr - 3 (Y empties), Gr - 1 from X into the emptied Y (refill), Gr - 1 again, then nothing.
    ``gangs``: the last two requests and one more form a gang that takes Gr - 1, fails and gives it back; a last gang takes it.
    Returns (rows, quirks, node_off, occ, req, gang_off)."""
    Gr = hi - lo
    W1 = ((Gr + 31) // 32 + 31) // 32
    assert Gr % 1024 >= 3 and W1 > 64
    flip = policy == E.POLICY_RIGHT_TO_LEFT
    occ = np.full(G, 0xFF, dtype=np.uint8)
    for x in (5, 40 * 1024 + 17, (W1 - 10) * 1024 + 100, Gr - 3):
        place_at(occ, lo, hi, flip, x, Y_BYTE)
    place_at(occ, lo, hi, flip, 9, Z_BYTE)
    place_at(occ, lo, hi, flip, Gr - 1, X_BYTE)
    n = 10 if gangs else 9
    req = W.alloc_requests(np.zeros(n, dtype=np.uint8))
    off = np.array([0, 2, 4, 6, 9, 10] if gangs else range(n + 1), dtype=np.uint32)
    return t16x8(), E.QUIRKS_REF_EXACT, eight_gpu_nodes(G), occ, req, off


ABORT_P = 7                         # T16mix-2 profile 7: size 8 at start 0 (FIXED quirks) — only an empty GPU admits it


def abort_call(G, lo, hi, policy):
    """T16mix-2, FIXED quirks, background 0x01 (no room for profile 7).  Storage-local: empty GPUs at 3, 50 K + 3 and 400 K + 3, a full
    one at 900 K + 3.  Gang 1 is profile 7 four times: it takes the three empty GPUs (the next one found in windows 1 and 10, then the
    class empties) and fails; the abort gives them back — the empty class's minimum restored to each, and the full class's minimum walked
    from 3 to 900 K + 3 (window 28).  Gang 2 (three times) takes them again; gangs 3 and 4 find nothing.
    Returns (rows, quirks, node_off, occ, req, gang_off)."""
    Gr = hi - lo
    assert Gr > 900 * 1024 + 3
    flip = policy == E.POLICY_RIGHT_TO_LEFT
    occ = np.full(G, 0x01, dtype=np.uint8)
    for x in (3, 50 * 1024 + 3, 400 * 1024 + 3):
        place_at(occ, lo, hi, flip, x, 0x00)
    place_at(occ, lo, hi, flip, 900 * 1024 + 3, 0xFF)
    req = W.alloc_requests(np.full(9, ABORT_P, dtype=np.uint8))
    return t16mix(2), E.QUIRKS_FIXED, eight_gpu_nodes(G), occ, req, np.array([0, 4, 7, 8, 9], dtype=np.uint32)


def live_call(rng, G=16384, n=2000):
    """T8tab, FIXED quirks, eight-GPU nodes on tables 0..7 in turn; on every table the first 256 GPUs hold every byte once, the rest
    whole bytes.  Returns (rows, node_off, node_table, occ, req)."""
    node_off = eight_gpu_nodes(G)
    n_nodes = len(node_off) - 1
    node_table = (np.arange(n_nodes) % 8).astype(np.uint8)
    occ = whole_bytes(rng, G)
    gtab = np.repeat(node_table, 8)
    for t in range(8):
        g = np.flatnonzero(gtab == t)[:256]
        occ[g] = (rng.next(256).argsort() % 256).astype(np.uint8)
    return t8tab(), node_off, node_table, occ, gang_call(rng, G, 16, n)


# (name, G, lo, hi, fixture): the shared / global memory switch of the class bitmaps
SWITCH_CASES = [("whole_4096", 4096, 0, 4096, "t16x8"), ("whole_4097", 4097, 0, 4097, "t16x8"),
                ("part_4096", TOP, 333333, 333333 + 4096, "t16x8"), ("part_4097", TOP, 333333, 333333 + 4097, "t16x8"),
                ("tables_4096", 4096, 0, 4096, "t8tab")]
SWITCH_SMEM = {"whole_4096": True, "whole_4097": False, "part_4096": True, "part_4097": False, "tables_4096": False}


def switch_call(rng, case, n):
    """(rows, quirks, node_off, node_table, occ, req, lo, hi) of a SWITCH_CASES entry."""
    name, G, lo, hi, fixture = case
    rows = FIXTURES[fixture]()
    node_off = eight_gpu_nodes(G)
    node_table = (rng.next(len(node_off) - 1) % np.uint64(8)).astype(np.uint8) if rows.ndim == 2 else None
    quirks = E.QUIRKS_FIXED if rows.ndim == 2 else E.QUIRKS_REF_EXACT
    req = gang_call(rng, G, rows.shape[-1], n)
    return rows, quirks, node_off, node_table, whole_bytes(rng, G), req, lo, hi


HALF = 1 << 19


def tie_call(G=TOP):
    """T16x8, background 0xFF: X (two free slots) at 3, Z (slot 7 free) at 2^19 - 1, Y (slot 1 free) at 2^19, 2^19 + 1 and 2^20 - 2.
    Nine ALLOCs of profile 0.  Best-fit: score 0 for Y and Z, so 2^19 - 1 beats 2^19 on the tie; min-frag: 16 pairs everywhere, so 3
    first, then the same tie.  Returns (rows, quirks, node_off, occ, req)."""
    occ = np.full(G, 0xFF, dtype=np.uint8)
    occ[3] = X_BYTE
    occ[HALF - 1] = Z_BYTE
    occ[[HALF, HALF + 1, G - 2]] = Y_BYTE
    return t16x8(), E.QUIRKS_REF_EXACT, eight_gpu_nodes(G), occ, W.alloc_requests(np.zeros(9, dtype=np.uint8))


def only_top_call(G=TOP):
    """T16x8, every GPU full but GPU 2^20 - 1 (slot 4 free); three ALLOCs of profile 0."""
    occ = np.full(G, 0xFF, dtype=np.uint8)
    occ[G - 1] = 0xEF
    return t16x8(), E.QUIRKS_REF_EXACT, eight_gpu_nodes(G), occ, W.alloc_requests(np.zeros(3, dtype=np.uint8))


def top_call(rng, name, G=TOP, n=300):
    """T16top or T16straddle, FIXED quirks: every GPU empty, slice 0 busy, slices 0 and 7 busy, or full; one ALLOC in three profile 15."""
    kinds = np.array([0x00, 0x01, 0x81, 0xFF], dtype=np.uint8)
    occ = kinds[(rng.next(G) % np.uint64(4)).astype(np.int64)]
    prof = (rng.next(n) % np.uint64(15)).astype(np.uint8)
    prof[rng.next(n) % np.uint64(3) == 0] = 15
    return FIXTURES[name](), E.QUIRKS_FIXED, eight_gpu_nodes(G), occ, W.alloc_requests(prof)


def lower_half_full(rng, G=TOP, n=400):
    """T8tab, FIXED quirks, eight-GPU nodes on random tables: the lower half full but for what the call's FREEs release, the upper half
    dense whole bytes; gang_call's mix.  Returns (rows, node_off, node_table, occ, req)."""
    node_off = eight_gpu_nodes(G)
    node_table = (rng.next(len(node_off) - 1) % np.uint64(8)).astype(np.uint8)
    occ = whole_bytes(rng, G, dense=True)
    occ[:G // 2] = 0xFF
    return t8tab(), node_off, node_table, occ, gang_call(rng, G, 16, n)


# ---- the generators reach their edges --------------------------------------------------------------------------------------------------
def sparse_edges(walk, Gr):
    e = walk.edges
    return {"later_window": any(x[0] == "window" and x[1] >= 1 for x in e),
            "window_1": any(x[0] == "window" and x[1] == 1 for x in e),
            "partial_last": Gr % 1024 != 0 and any(x[0] == "window" and x[2] and x[3] for x in e),
            "inf_after_windows": any(x[0] == "inf" and x[1] >= 31 for x in e),
            "refill": ("refill",) in e}


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("where", ["whole", "partition"])
@pytest.mark.parametrize("gangs", [False, True], ids=["batch", "gangs"])
def test_sparse_call_reaches_every_branch_of_the_walk(policy, where, gangs):
    G, lo, hi = (SPARSE_G, 0, SPARSE_G) if where == "whole" else (TOP, SPARSE_LO, TOP)
    rows, quirks, node_off, occ, req, off = sparse_call(G, lo, hi, policy, gangs)
    out, _after, walk = replay(node_off, rows, occ, req, off, quirks, policy, lo=lo, hi=hi)
    assert all(sparse_edges(walk, hi - lo).values()), sparse_edges(walk, hi - lo)
    st = out["status"].tolist()
    if gangs:
        assert st == [E.ST_PLACED] * 6 + [E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_GANG_ABORTED, E.ST_PLACED]
        assert out["gpu"][9] == out["gpu"][5] and ("restore", INF) in walk.edges
    else:
        assert st == [E.ST_PLACED] * 7 + [E.ST_NO_CAPACITY] * 2
        assert out["gpu"][5] == out["gpu"][6]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("where", ["whole", "partition"])
def test_abort_call_puts_far_minima_back(policy, where):
    G, lo, hi = (SPARSE_G, 0, SPARSE_G) if where == "whole" else (TOP, SPARSE_LO, TOP)
    rows, quirks, node_off, occ, req, off = abort_call(G, lo, hi, policy)
    out, after, walk = replay(node_off, rows, occ, req, off, quirks, policy, lo=lo, hi=hi)
    st = out["status"].tolist()
    assert st == [E.ST_GANG_ABORTED] * 3 + [E.ST_NO_CAPACITY] + [E.ST_PLACED] * 3 + [E.ST_NO_CAPACITY] * 2
    empty = sorted(int(g) for g in np.flatnonzero(occ == 0))
    assert sorted(int(g) for g in out["gpu"][4:7]) == empty and (after[empty] == 0xFF).all()
    restores = [x[1] for x in walk.edges if x[0] == "restore"]
    assert restores == [INF, 350, 50], restores                     # each member back below a minimum a window or more above it
    assert ("abort_min",) in walk.edges and ("window", 28, False, False) in walk.edges
    # without the abort the second gang would find nothing: the three GPUs are the only room
    solo, _ = BF.place(node_off, rows, after, req[:3], quirks, policy, lo=lo, hi=hi)
    assert (solo["status"] == E.ST_NO_CAPACITY).all()


def test_live_call_populates_all_2048_classes():
    rng = W.SplitMix64(2048)
    rows, node_off, node_table, occ, req = live_call(rng)
    gtab = np.repeat(node_table, 8).astype(np.int64)
    assert len(np.unique(gtab * 256 + occ)) == 8 * 256
    for policy in BF_POLICIES:
        out, _ = BF.place(node_off, rows, occ, req[:600], E.QUIRKS_FIXED, policy, node_table)
        placed = out[out["status"] == E.ST_PLACED]
        assert len(set(gtab[placed["gpu"]].tolist())) == 8


@pytest.mark.parametrize("case", SWITCH_CASES, ids=[c[0] for c in SWITCH_CASES])
def test_switch_cases_sit_on_both_sides_of_the_shared_memory_switch(case):
    rng = W.SplitMix64(4096)
    rows, quirks, node_off, node_table, occ, req, lo, hi = switch_call(rng, case, 50)
    n_tables = 1 if rows.ndim == 1 else 8
    assert bitmaps_in_smem(n_tables, hi - lo) == SWITCH_SMEM[case[0]]
    if case[0].startswith("part"):
        assert lo % 32 != 0 and hi <= TOP
    if SWITCH_SMEM[case[0]]:
        stride = (hi - lo + 31) // 32 + ((hi - lo + 31) // 32 + 31) // 32
        assert 256 * stride * 4 == 132 * 1024               # the shared memory k_bestfit asks for at 4 096 GPUs
    out, _ = BF.place(node_off, rows, occ, req, quirks, E.POLICY_BEST_FIT, node_table, lo, hi)
    assert (out["status"] == E.ST_PLACED).any()


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_tie_call_breaks_ties_across_2_19(policy):
    rows, quirks, node_off, occ, req = tie_call()
    out, _, _walk = replay(node_off, rows, occ, req, np.arange(len(req) + 1), quirks, policy)     # every pick is its class minimum
    gpus = [int(g) for g in out["gpu"][:8]]
    assert gpus.index(HALF - 1) < gpus.index(HALF) < gpus.index(HALF + 1) < gpus.index(TOP - 2)
    # the GPU below 2^19 and those above tie on the score, in different classes
    mf = min_frag_scores(rows, quirks)[0]
    assert mf[Z_BYTE] == mf[Y_BYTE] == mf[X_BYTE] == 16 and bin(Z_BYTE).count("1") == bin(Y_BYTE).count("1")
    if policy == E.POLICY_BEST_FIT:
        assert gpus[:4] == [HALF - 1, HALF, HALF + 1, TOP - 2] and gpus[4:6] == [3, 3]
    else:
        assert gpus[:2] == [3, 3] and gpus[2:6] == [HALF - 1, HALF, HALF + 1, TOP - 2]
    assert out["status"][8] == E.ST_NO_CAPACITY


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_only_top_call_places_on_the_last_gpu(policy):
    rows, quirks, node_off, occ, req = only_top_call()
    out, after = BF.place(node_off, rows, occ, req, quirks, policy)
    assert out["gpu"][0] == TOP - 1 and out["status"].tolist() == [E.ST_PLACED, E.ST_NO_CAPACITY, E.ST_NO_CAPACITY]
    assert after[TOP - 1] == 0xFF


@pytest.mark.parametrize("name", ["t16top", "t16straddle"])
def test_top_call_reaches_min_frag_scores_above_63(name):
    rng = W.SplitMix64(63)
    rows, quirks, node_off, occ, req = top_call(rng, name, G=1 << 14)
    score = min_frag_scores(rows, quirks)[15]
    out, _ = BF.place(node_off, rows, occ, req, quirks, E.POLICY_MIN_FRAG)
    won = out[(req["profile"] == 15) & (out["status"] == E.ST_PLACED)]
    assert len(won)
    fits = np.flatnonzero(score[occ] > 0)
    seen = set(score[occ[fits]].tolist())
    assert max(seen) > 63
    if name == "t16straddle":
        # both sides of 64 compete for profile 15: a key that kept only the low 6 bits of the score would pick another GPU
        assert min(seen) < 64
        assert np.argmin(score[occ[fits]] * (1 << 24) + fits) != np.argmin((score[occ[fits]] & 63) * (1 << 24) + fits)


def test_lower_half_full_places_above_2_19_only_through_frees():
    rng = W.SplitMix64(19)
    rows, node_off, node_table, occ, req = lower_half_full(rng, G=1 << 14)
    out, _ = BF.place_gangs(node_off, rows, occ, req, small_gangs(rng, len(req)), E.QUIRKS_FIXED, E.POLICY_BEST_FIT, node_table)
    placed = out[(out["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)]
    assert (placed["gpu"] >= (1 << 13)).any() and (out["status"] == E.ST_GANG_ABORTED).any()


# ---- the checker, pinned -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_checker_equals_ref_fast_and_the_range_restatement(name, quirks, policy):
    """Whole inventories against oracle.Fast, cut ranges against range_oracle.place_range: records and the whole occupancy."""
    rows = FIXTURES[name]()
    rng = W.SplitMix64(9000 + 10 * quirks + 100 * policy + len(name))
    for trial in range(4):
        node_off, node_table, occ = cluster(rng, rows, 40 + int(rng.next1() % 40))
        G = int(node_off[-1])
        req = gang_call(rng, G, rows.shape[-1], 200)
        if trial % 2 == 0:
            ref = oracle.Fast(node_off, rows, quirks, policy, node_table=node_table)
            ref.load(occ)
            want, want_occ = ref.place(req), ref.occupancy()
            lo, hi = 0, G
        else:
            lo, hi = 1 + int(rng.next1() % (G // 3)), G - 1 - int(rng.next1() % (G // 3))
            want, want_occ = RO.place_range(node_off, rows, occ, lo, hi, req, quirks, policy, node_table)
        got, got_occ = BF.place(node_off, rows, occ, req, quirks, policy, node_table, lo, hi)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (trial, bad[:4], got[bad[:4]], want[bad[:4]])
        assert np.array_equal(got_occ, want_occ), trial


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_checker_equals_gang_oracle(name, quirks, policy):
    """Gangs of every shape, whole inventories and cut partitions, against gang_oracle.fast_place_gangs over oracle.Fast / RangeFast."""
    rows = FIXTURES[name]()
    rng = W.SplitMix64(9500 + 10 * quirks + 100 * policy + len(name))
    outcomes = set()
    for trial, kind in enumerate(GANG_SHAPES):
        node_off, node_table, occ = cluster(rng, rows, 40 + int(rng.next1() % 40))
        G = int(node_off[-1])
        occ = whole_bytes(rng, G, dense=True)
        lo, hi = (0, G) if trial % 2 == 0 else (1 + int(rng.next1() % (G // 3)), G - 1 - int(rng.next1() % (G // 3)))
        n = 130 if kind == "straddle" else 100
        req = gang_call(rng, G, rows.shape[-1], n)
        off = gang_offsets(rng, kind, n)
        if (lo, hi) == (0, G):
            ref = oracle.Fast(node_off, rows, quirks, policy, node_table=node_table)
            ref.load(occ)
        else:
            ref = RO.RangeFast(node_off, rows, occ, lo, hi, quirks, policy, node_table)
        want = GO.fast_place_gangs(ref, req, off, gang_sizes(rows, node_table))
        got, got_occ = BF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (kind, bad[:4], got[bad[:4]], want[bad[:4]])
        assert np.array_equal(got_occ, ref.occupancy()), kind
        outcomes |= set(np.unique(got["status"]).tolist())
    assert {E.ST_PLACED, E.ST_GANG_ABORTED} <= outcomes


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name", ["t8tab", "t16top", "t16straddle", "t16mix2"])
def test_memo_on_equals_memo_off(name, policy):
    rows = FIXTURES[name]()
    quirks = 1 if name == "t16mix2" else E.QUIRKS_FIXED
    rng = W.SplitMix64(4100 + policy + len(name))
    for G in (64, 777):
        node_off = eight_gpu_nodes(G)
        node_table = (rng.next(len(node_off) - 1) % np.uint64(8)).astype(np.uint8) if rows.ndim == 2 else None
        occ = whole_bytes(rng, G)
        req = gang_call(rng, G, rows.shape[-1], 300)
        off = gang_offsets(rng, "mixed", 300)
        a = BF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, 3, G - 2, memo=True)
        b = BF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, 3, G - 2, memo=False)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), G
        assert (a[0]["status"] == E.ST_PLACED).any()


def test_min_frag_at_2_20_gpus_takes_seconds():
    """A MIN_FRAG batch of 400 requests over 2^20 GPUs on T8tab with node tables: each ALLOC scans every GPU.  Measured on one core of
    an Intel Xeon server CPU: 1.1-1.3 s with the memo, 6.6 s with it off; the bound leaves room for slower machines."""
    rng = W.SplitMix64(TOP)
    rows, node_off, node_table, occ, req = lower_half_full(rng)
    t0 = time.perf_counter()
    out, _ = BF.place(node_off, rows, occ, req, E.QUIRKS_FIXED, E.POLICY_MIN_FRAG, node_table)
    assert time.perf_counter() - t0 < 20
    assert (out["gpu"][out["status"] == E.ST_PLACED] >= HALF).any()
