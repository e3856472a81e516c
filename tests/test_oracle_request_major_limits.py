"""Gangs, preemption and node scoring at the profile-table limits of the ABI — the generators, their self-checks and the pins of the
checkers at these shapes (CPU only).  ``test_gpu_request_major_limits.py`` runs the same inputs through k_bestfit<.., kGang = true>,
k_victim_map + k_preempt and k_nodefit.

The fixtures are those of ``test_oracle_table_limits.py`` (T16x8, T16mix-1/2, T8tab with its node tables).  Built here:
  fixture_tables   the fixture rows as Migplacement rows (names "p<index>"), for the restatements on custom-resource dicts
  whole_bytes      occupancy of whole bytes (slice 7 busy as often as slice 0), some GPUs empty and some full
  gang_call        ALLOCs of every name and an unknown one, FREEs (some malformed), NOOPs; gangs of one, mixed gangs, one gang that
                   straddles 32-request blocks, one gang that is the whole call
  p15_call         a nearly full inventory and gangs of profile 15: one that takes every place profile 15 has plus one (it aborts with
                   profile 15 dead inside it), then gangs that place profile 15 again (bit 15 of the dead mask was restored)
  preempt_state    per GPU one kind: empty, pinned, eight one-slice victims of priority b or b + 1 (equal highest priorities and sums
                   one apart compete for a size-8 preemptor), spans of every size 1..8 (victims or pinned), one size-8 victim, eight victims of priority 254
  preemptors       every name and an unknown one, priorities 0, 254, 255 and a few in between
  scoring_nodes    ragged nodes with empty ones; at the top exactly the 2^20 nodes a node-scoring engine accepts
"""
import os
import random
import re

import numpy as np
import pytest

import oracle
from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W

import gang_oracle as GO
import node_score_fast as NF
import node_score_oracle as NO
import preempt_fast as PF
import preempt_oracle as PO
from test_oracle_table_limits import candidate_mask, t16mix, t16x8, t8tab, t8tab_node_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUIRKS2 = (E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED)
FIXTURES = {"t16x8": t16x8, "t16mix1": lambda: t16mix(1), "t16mix2": lambda: t16mix(2), "t8tab": t8tab}
TOP_NODES = 1 << 20                 # node scoring: isl_load_inventory's node limit (include/islplace.h, rule 7)


# ---- the fixtures as custom-resource rows -------------------------------------------------------------------------------------------
def tables2(rows):
    return rows if rows.ndim == 2 else rows[None]


def names_of(rows):
    return ["p%d" % p for p in range(rows.shape[-1])]


def fixture_tables(rows):
    """Every table of [P] or [T][P] rows as tables.py rows (name, size, starts, GI id); a name a table does not know has no row."""
    return [[("p%d" % p, int(r["size"]), [int(s) for s in r["starts"][:r["n_starts"]]], int(r["gi"])) for p, r in enumerate(tab)
             if r["n_starts"]] for tab in tables2(rows)]


def fixture_migplacement(rows):
    return [tables.migplacement(t) for t in fixture_tables(rows)]


def gpu_tables(node_off, node_table):
    return np.repeat(np.asarray(node_table, dtype=np.uint8), np.diff(np.asarray(node_off, dtype=np.int64)))


def node_tables_for(rows, rng, n_nodes):
    return t8tab_node_tables(rng, n_nodes) if rows.ndim == 2 else None


# ---- occupancy, nodes -----------------------------------------------------------------------------------------------------------------
def whole_bytes(rng, G, dense=False):
    """SplitMix64 occupancy over all 8 slices; about 1/16 of the GPUs empty and 1/16 full."""
    a, b = rng.next(G), rng.next(G)
    occ = ((a | b) if dense else (a & b)) & np.uint64(0xFF)
    kind = rng.next(G) % np.uint64(16)
    occ[kind == 0] = 0
    occ[kind == 1] = 0xFF
    return occ.astype(np.uint8)


def scoring_nodes(rng, n_nodes, max_gpus=8, empty_share=8):
    """Offsets of n_nodes nodes of 1..max_gpus GPUs, about one in ``empty_share`` empty (never the last)."""
    sizes = 1 + (rng.next(n_nodes) % np.uint64(max_gpus)).astype(np.int64)
    sizes[rng.next(n_nodes) % np.uint64(empty_share) == 0] = 0
    sizes[-1] = max(1, sizes[-1])
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


def top_nodes(rng, extra=0):
    """TOP_NODES + extra nodes of 0..1 GPUs (about one in eight empty) over at most 2^20 GPUs: the largest inventory a node-scoring
    engine accepts (extra = 0: five full levels of 32-ary score trees) and, with extra = 1, the smallest it refuses."""
    return scoring_nodes(rng, TOP_NODES + extra, max_gpus=1)


def planner_levels(n_nodes):
    """The level counts run_nodefit (islplace.cu) plans for a range of n_nodes nodes: one per level down to the root."""
    out, cnt = [], n_nodes
    while True:
        out.append(cnt)
        if cnt == 1:
            return out
        cnt = (cnt + 31) // 32


# ---- gangs -----------------------------------------------------------------------------------------------------------------------
def gang_call(rng, G, n_names, n):
    req = W.alloc_requests((rng.next(n) % np.uint64(n_names + 1)).astype(np.uint8))
    req["profile"][req["profile"] == n_names] = E.PROFILE_UNKNOWN
    for i in np.flatnonzero(rng.next(n) % np.uint64(11) == 0):
        g = int(rng.next1() % (G + 2))                  # G, G + 1: BAD_SPAN
        start = int(rng.next1() % 8)
        req[i] = (g, 0, E.OP_FREE, start, 1 + int(rng.next1() % (8 - start)))
    req["op"][rng.next(n) % np.uint64(29) == 0] = E.OP_NOOP
    return req


GANG_SHAPES = ("ones", "mixed", "straddle", "whole")


def gang_offsets(rng, kind, n):
    if kind == "ones":
        return np.arange(n + 1, dtype=np.uint32)
    if kind == "whole":
        return np.array([0, n], dtype=np.uint32)
    off = [0]
    if kind == "straddle":                              # small gangs around one gang of 40..100 members across 32-request blocks
        off.append(5 + int(rng.next1() % 20))
        off.append(off[-1] + 40 + int(rng.next1() % 61))
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % 40)))
    return np.asarray(off, dtype=np.uint32)


def gang_sizes(rows, node_table):
    return GO.default_sizes(rows, node_table) if rows.ndim == 2 else GO.default_sizes(rows)


def p15_call(rng, rows, node_off, node_table, quirks):
    """(occupancy, requests, gang offsets): every GPU full but about 1/256 empty (1/8 with per-node tables, where only table 7 knows
    profile 15) and as many of random bytes; gang 1 is profile 15 as often as it fits plus once more, gang 2 is one request of another
    profile, gangs 3 and 4 are profile 15 once each."""
    G = int(node_off[-1])
    occ = np.full(G, 0xFF, dtype=np.uint8)
    kind = rng.next(G) % np.uint64(256 if rows.ndim == 1 else 8)
    occ[kind == 0] = 0
    occ[kind == 1] = (rng.next(int((kind == 1).sum())) & np.uint64(0xFF)).astype(np.uint8)
    probe = oracle.Fast(node_off, rows, quirks, node_table=node_table)
    probe.load(occ)
    room = int((probe.place(W.alloc_requests(np.full(8 * G, 15, dtype=np.uint8)))["status"] == E.ST_PLACED).sum())
    prof = [15] * (room + 1) + [int(rng.next1() % 15), 15, 15]
    return occ, W.alloc_requests(np.array(prof, dtype=np.uint8)), np.array([0, room + 1, room + 2, room + 3, room + 4], dtype=np.uint32)


# ---- preemption -------------------------------------------------------------------------------------------------------------------
EMPTY, PINNED, EIGHT, SPANS, WHOLE, EIGHT254 = range(6)
KIND_MIX = (0.0, 0.25, 0.3, 0.36, 0.05, 0.04)     # empty GPUs: a handful, whatever G (see preempt_state)
PREEMPTOR_PRIORITIES = np.array([0, 1, 8, 101, 200, 254, 254, 255, 255, 255])


def preempt_state(rng, G, mix=KIND_MIX, kinds=None):
    """(occupancy, victims in random order, kind of every GPU) from a numpy Generator; ``kinds`` overrides the draw.  Free room stays
    scarce at every G — two empty GPUs and a few free spans — so that most preemptors have to evict; the first and the last GPU
    hold the cheapest victims there are, one size-8 victim of priority 0 each."""
    if kinds is None:
        kinds = rng.choice(len(mix), G, p=mix)
        kinds[rng.integers(0, G, 2)] = EMPTY
        kinds[[0, -1]] = WHOLE
    free_share = min(0.15, 1.0 / max(1, int((kinds == SPANS).sum())))
    occ = np.zeros(G, dtype=np.uint8)
    occ[np.isin(kinds, (PINNED, EIGHT, WHOLE, EIGHT254))] = 0xFF
    parts = []                                          # (gpu, start, size, priority) columns

    def eight(g, pr):
        parts.append((np.repeat(g, 8), np.tile(np.arange(8), len(g)), np.ones(8 * len(g), np.int64), pr.reshape(-1)))

    g = np.flatnonzero(kinds == EIGHT)
    # b + 1 three times in four: few GPUs share the smallest sums, many the ones just above, where sums 2j and 2j + 1 compete
    eight(g, rng.choice(np.array([0, 7, 100, 253]), len(g))[:, None] + (rng.random((len(g), 8)) < 0.75))
    g = np.flatnonzero(kinds == EIGHT254)
    eight(g, np.full((len(g), 8), 254))
    g = np.flatnonzero(kinds == WHOLE)
    pr = rng.integers(9, 255, len(g))                   # above every priority of an eight-victim GPU of base 0 ...
    pr[[0, -1][:len(g)]] = 0                            # ... but the first and the last in canonical order: the cheapest there is
    parts.append((g, np.zeros(len(g), np.int64), np.full(len(g), 8), pr))
    g = np.flatnonzero(kinds == SPANS)
    pos = np.zeros(len(g), dtype=np.int64)
    while True:
        live = np.flatnonzero(pos < 8)
        if len(live) == 0:
            break
        size = np.minimum(rng.integers(1, 9, len(live)), 8 - pos[live])
        busy = rng.random(len(live)) >= free_share
        listed = busy & (rng.random(len(live)) < 0.7)
        gg, ss = g[live], pos[live]
        occ[gg[busy]] |= (((1 << size[busy]) - 1) << ss[busy]).astype(np.uint8)
        low = rng.random(len(live)) < 0.5
        pr = np.where(low, rng.integers(3, 8, len(live)), rng.integers(3, 255, len(live)))     # above eight-victim GPUs of base 0
        parts.append((gg[listed], ss[listed], size[listed], pr[listed]))
        pos[live] += size
    vic = np.zeros(sum(len(p[0]) for p in parts), dtype=E.VICTIM_DTYPE)
    for field, k in (("gpu", 0), ("start", 1), ("size", 2), ("priority", 3)):
        vic[field] = np.concatenate([p[k] for p in parts])
    return occ, vic[rng.permutation(len(vic))], kinds


def preemptors(rng, n, n_names):
    req = np.zeros(n, dtype=E.REQUEST_DTYPE)
    req["handle"] = np.arange(n)
    req["profile"] = rng.integers(0, n_names, n)
    req["op"] = E.OP_ALLOC
    odd = rng.random(n) < 0.03                          # unknown profiles and NOOPs are answered in place
    req["profile"][odd & (rng.random(n) < 0.5)] = E.PROFILE_UNKNOWN
    req["op"][odd & (req["profile"] != E.PROFILE_UNKNOWN)] = E.OP_NOOP
    return req, rng.choice(PREEMPTOR_PRIORITIES, n).astype(np.uint8)


def preemptors_for(rng, rows, n):
    """``preemptors``, a quarter of them turned into ALLOCs of the biggest profile when a row of the fixture covers all 8 slices: those
    take empty GPUs, then size-8 victims, then eight victims at once."""
    req, prio = preemptors(rng, n, rows.shape[-1])
    p = biggest_profile(rows)
    if tables2(rows)["size"][:, p].max() == 8:
        big = rng.random(n) < 0.25
        req["profile"][big], req["op"][big] = p, E.OP_ALLOC
    return req, prio


def biggest_profile(rows):
    """The profile name of the largest size any table gives it (T16mix-2: profile 7, size 8)."""
    sizes = tables2(rows)["size"] * (tables2(rows)["n_starts"] > 0)
    return int(np.argmax(sizes.max(axis=0)))


def top_partition_case(rng, rows, G, lo, n):
    """The top partition [lo, G): pinned GPUs, a few empty ones, eight-victim GPUs (some all 254) and size-8 victims; preemptors mostly
    of the biggest profile at priority 255, so that they run through everything cheaper and then evict eight victims of priority 254."""
    kinds = np.full(G, PINNED)
    kinds[lo:] = rng.choice(6, G - lo, p=(0.02, 0.6, 0.08, 0.0, 0.1, 0.2))
    occ, vic, kinds = preempt_state(rng, G, kinds=kinds)
    req, prio = preemptors(rng, n, rows.shape[-1])
    big = rng.random(n) < 0.6
    req["profile"][big], req["op"][big], prio[big] = biggest_profile(rows), E.OP_ALLOC, 255
    return occ, vic, req, prio


def sm_limit_gpus(sms):
    """The G at which k_preempt runs one CTA per SM and the last CTA owns a single GPU (isl_preempt's grid: min(SMs, ceil(G / 512))
    CTAs of ceil(G / grid) GPUs)."""
    return (sms - 1) * 512 + 1


def winner_stats(vic, evict, out):
    """Per PLACED preemptor: (number of victims, their priority sum, largest victim size)."""
    st = []
    for r, row in zip(out, evict):
        if r["status"] == E.ST_PLACED:
            ks = [int(k) for k in row if k != E.GPU_NONE]
            st.append((len(ks), int(vic["priority"][ks].astype(np.int64).sum()) if ks else 0, max((int(vic["size"][k]) for k in ks), default=0)))
    return st


def row_positions(rows, node_table_of_gpu, req, out):
    """Position in its row of every PLACED record's start."""
    r2 = tables2(rows)
    pos = []
    for q, r in zip(req, out):
        if r["status"] == E.ST_PLACED:
            row = r2[int(node_table_of_gpu[int(r["gpu"])]), int(q["profile"])]
            pos.append(list(row["starts"][:row["n_starts"]]).index(int(r["start"])))
    return pos


# ---- custom-resource dicts --------------------------------------------------------------------------------------------------------
def scoring_items(node_off, occ, rows, node_table):
    """One Instaslice object per node, its own Migplacement, GPUs named so that sorted UUID = canonical order, busy slices dangling."""
    migs = fixture_migplacement(rows)
    items = []
    for n in range(len(node_off) - 1):
        gs = range(int(node_off[n]), int(node_off[n + 1]))
        prepared = {"p%d-%d" % (g, x): {"parent": "GPU-%07d" % g, "start": x, "size": 1, "podUUID": ""}
                    for g in gs for x in range(8) if int(occ[g]) >> x & 1}
        items.append({"metadata": {"name": "node-%d" % n},
                      "spec": {"MigGPUUUID": {"GPU-%07d" % g: "" for g in gs}, "migplacement": migs[0 if node_table is None else int(node_table[n])],
                               "prepared": prepared, "allocations": {}}})
    return items


def preempt_items(node_off, occ, rows, node_table, vic):
    """The same objects with victim k an Allocations entry "v<k>" and every other busy slice a dangling Prepared slice."""
    items = scoring_items(node_off, np.zeros_like(occ), rows, node_table)
    covered = np.zeros(len(occ), dtype=np.int64)
    for k, v in enumerate(vic):
        g = int(v["gpu"])
        n = int(np.searchsorted(node_off, g, side="right")) - 1
        items[n]["spec"]["allocations"]["v%d" % k] = {"gpuUUID": "GPU-%07d" % g, "start": int(v["start"]), "size": int(v["size"]),
                                                      "allocationStatus": "created"}
        covered[g] |= PO.span(v["start"], v["size"])
    for g in range(len(occ)):
        n = int(np.searchsorted(node_off, g, side="right")) - 1
        for x in range(8):
            if (int(occ[g]) & ~int(covered[g])) >> x & 1:
                items[n]["spec"]["prepared"]["p%d-%d" % (g, x)] = {"parent": "GPU-%07d" % g, "start": x, "size": 1, "podUUID": ""}
    return items


# ---- self-checks of the generators --------------------------------------------------------------------------------------------------
def test_fixture_migplacement_round_trips():
    for name, make in FIXTURES.items():
        rows = make()
        for t, mig in enumerate(fixture_migplacement(rows)):
            back, index = ctl.profile_rows(mig)
            for p in range(rows.shape[-1]):
                want = tables2(rows)[t, p]
                if not want["n_starts"]:
                    assert "p%d" % p not in index, (name, t, p)
                    continue
                got = back[index["p%d" % p]]
                assert (got["size"], got["n_starts"], list(got["starts"])) == (want["size"], want["n_starts"], list(want["starts"])), (name, t, p)


def test_widths_of_the_fixtures():
    """Rule 2's width (largest start + size over a table's rows, illegal starts included): T16mix-2 is wider than 8, T8tab has 8 tables
    of which not all share one width, and some table lacks a name."""
    def widths(rows):
        r2 = tables2(rows)
        return [max(int(s) + int(r["size"]) for r in tab for s in r["starts"][:r["n_starts"]]) for tab in r2]
    assert widths(t16x8()) == [8]
    assert widths(t16mix(2)) == [10]
    w8 = widths(t8tab())
    assert len(w8) == 8 and len(set(w8)) > 1 and max(w8) > 8, w8
    assert (t8tab()["n_starts"] == 0).any(axis=1).all()


def test_whole_bytes_reach_slice_7_and_both_ends():
    occ = whole_bytes(W.SplitMix64(1), 4097)
    assert (occ & 0x80).any() and (occ == 0).any() and (occ == 0xFF).any()
    assert ((occ & 0x80) != 0).mean() > 0.15


def test_planner_needs_a_sixth_level_beyond_2_20_nodes():
    """The node limit of a node-scoring engine, restated: run_nodefit's level plan fits kNfMaxLevels levels for up to kNfMaxNodes nodes,
    empty nodes included, and needs one more for a single node beyond (1 048 577 -> 32 769 -> 1 025 -> 33 -> 2 -> 1).  The device
    test loads top_nodes(rng) (accepted) and top_nodes(rng, 1) (ISL_ERANGE)."""
    src = open(os.path.join(ROOT, "instaslice_b200", "csrc", "isl_kernels.cuh")).read()
    max_levels = int(re.search(r"kNfMaxLevels = (\d+);", src).group(1))
    max_nodes = 1 << int(re.search(r"kNfMaxNodes = 1u << (\d+);", src).group(1))
    assert max_nodes == TOP_NODES == E.NODE_SCORING_MAX_NODES
    assert planner_levels(TOP_NODES) == [1 << 20, 1 << 15, 1 << 10, 32, 1] and len(planner_levels(TOP_NODES)) == max_levels
    assert planner_levels(TOP_NODES + 1) == [1048577, 32769, 1025, 33, 2, 1]
    assert len(planner_levels(TOP_NODES + 1)) == max_levels + 1
    header = open(os.path.join(ROOT, "include", "islplace.h")).read()
    assert "isl_load_inventory: ISL_ERANGE for more than 2^20 nodes" in header
    rng = W.SplitMix64(20)
    node_off = top_nodes(rng)
    sizes = np.diff(node_off.astype(np.int64))
    assert len(sizes) == TOP_NODES and int(node_off[-1]) <= 1 << 20 and (sizes == 0).any() and sizes[-1] == 1
    assert len(top_nodes(rng, 1)) - 1 == TOP_NODES + 1 and int(top_nodes(rng, 1)[-1]) <= 1 << 20


def test_p15_call_aborts_with_profile_15_dead_and_places_it_after():
    for name in ("t16x8", "t8tab"):
        rows = FIXTURES[name]()
        rng = W.SplitMix64(15)
        node_off = eight_gpu_nodes(4097)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        occ, req, off = p15_call(rng, rows, node_off, node_table, E.QUIRKS_FIXED)
        ref = oracle.Fast(node_off, rows, E.QUIRKS_FIXED, node_table=node_table)
        ref.load(occ)
        out = GO.fast_place_gangs(ref, req, off, gang_sizes(rows, node_table))
        room = int(off[1]) - 1
        assert room >= 32, (name, room)                                     # gang 1 straddles 32-request blocks
        assert (out["status"][:room] == E.ST_GANG_ABORTED).all() and out["status"][room] == E.ST_NO_CAPACITY
        assert out["status"][room + 2] == E.ST_PLACED and int(out["gpu"][room + 2]) != E.GPU_NONE
        # gang 1 placed profile 15 room times before it failed: ref_fast's per-request placement agrees
        probe = oracle.Fast(node_off, rows, E.QUIRKS_FIXED, node_table=node_table)
        probe.load(occ)
        assert (probe.place(req[:room + 1])["status"][:room] == E.ST_PLACED).all()


def eight_gpu_nodes(G):
    """G GPUs in nodes of 8 (the last one smaller when G is not a multiple of 8)."""
    off = list(range(0, G, 8)) + [G]
    return np.asarray(off, dtype=np.uint32)


def test_gang_shapes():
    rng = W.SplitMix64(3)
    for n in (300, 2500):
        off = gang_offsets(rng, "straddle", n)
        big = int(np.diff(off.astype(np.int64)).max())
        assert big >= 40 and off[-1] == n
        a = int(np.flatnonzero(np.diff(off.astype(np.int64)) == big)[0])
        assert int(off[a]) // 32 != (int(off[a + 1]) - 1) // 32


@pytest.mark.parametrize("name,quirks", [("t16x8", E.QUIRKS_REF_EXACT), ("t16mix2", E.QUIRKS_FIXED), ("t8tab", E.QUIRKS_FIXED)])
def test_preempt_generator_reaches_the_key_limits(name, quirks):
    """On the inputs the device test uses at the SM-count G: spans of every size, every victim and preemptor priority class, a size-8
    victim evicted, eight victims evicted at once, the last position of an 8-start row (T16x8)."""
    rows = FIXTURES[name]()
    rng = np.random.default_rng(7)
    G = sm_limit_gpus(132) // 8                          # a smaller inventory of the same generator
    node_off = eight_gpu_nodes(G)
    node_table = t8tab_node_tables(W.SplitMix64(8), len(node_off) - 1) if rows.ndim == 2 else None
    occ, vic, kinds = preempt_state(rng, G)
    req, prio = preemptors_for(rng, rows, 400)
    assert set(vic["size"].tolist()) == set(range(1, 9))
    assert int(vic["priority"].max()) == 254 and int(vic["priority"].min()) == 0
    assert {0, 254, 255} <= set(prio.tolist())
    rc, out, evict = PF.preempt(node_off, rows, occ, req, prio, vic, quirks, E.POLICY_FIRST_FIT, node_table)
    assert rc == E.OK
    st = winner_stats(vic, evict, out)
    assert any(s[2] == 8 for s in st)                                       # a size-8 victim leaves
    if name == "t16x8":
        assert 7 in row_positions(rows, np.zeros(G, np.uint8), req, out)    # the last position of an 8-start row wins
    if name == "t16mix2":
        assert any(s[0] == 8 for s in st)                                   # eight one-slice victims at once


def test_top_partition_evicts_eight_victims_of_priority_254():
    """The top-partition case of the device test, on a smaller inventory with the same partition size: some winning V is eight victims
    of priority 254 (sum 2 032, the largest the key's 11-bit field holds)."""
    rows = t16mix(2)
    rng = np.random.default_rng(2032)
    G = 8192
    lo = G - 1000
    node_off = eight_gpu_nodes(G)
    occ, vic, req, prio = top_partition_case(rng, rows, G, lo, 400)
    rc, out, evict = PF.preempt(node_off, rows, occ, req, prio, vic, E.QUIRKS_FIXED, E.POLICY_BEST_FIT, lo=lo, hi=G)
    assert rc == E.OK
    st = winner_stats(vic, evict, out)
    assert (8, 2032, 1) in st
    assert any(s[2] == 8 for s in st)
    assert ((out["gpu"][out["status"] == E.ST_PLACED] >= lo)).all()


# ---- the checkers against each other at the limits ------------------------------------------------------------------------------
@pytest.mark.parametrize("quirks", QUIRKS2)
@pytest.mark.parametrize("name", ["t16mix2", "t8tab"])
def test_preempt_fast_agrees_with_preempt_oracle(name, quirks):
    rows = FIXTURES[name]()
    names = names_of(rows)
    rng = np.random.default_rng(100 + quirks + len(name))
    srng = W.SplitMix64(200 + quirks)
    for trial in range(6):
        n_nodes = 1 + int(srng.next1() % 12)
        node_off = W.node_offsets(n_nodes, 1) if trial == 0 else np.concatenate([[0], np.cumsum(1 + srng.next(n_nodes) % np.uint64(8))]).astype(np.uint32)
        G = int(node_off[-1])
        node_table = node_tables_for(rows, srng, n_nodes)
        occ, vic, _kinds = preempt_state(rng, G)
        req, prio = preemptors(rng, 40, rows.shape[-1])
        policy = (E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_BEST_FIT)[trial % 3]
        rc, out, evict = PF.preempt(node_off, rows, occ, req, prio, vic, quirks, policy, node_table)
        assert rc == E.OK
        items = preempt_items(node_off, occ, rows, node_table, vic)
        pods = [{"profile": names[q["profile"]] if q["profile"] < len(names) else "unknown", "rank": int(r)} for q, r in zip(req, prio)]
        live = req["op"] == E.OP_ALLOC
        got = PO.preempt_cr(items, [p for p, a in zip(pods, live) if a], {"v%d" % k: int(v["priority"]) for k, v in enumerate(vic)},
                            quirks, policy)
        for (kind, where, gone), r, row in zip(got, out[live], evict[live]):
            ks = sorted(int(k) for k in row if k != E.GPU_NONE)
            if r["status"] != E.ST_PLACED:
                assert kind == "none" and not ks, (trial, r)
                continue
            assert kind == ("preempt" if ks else "fits")
            assert (int(where["gpuUUID"][4:]), where["start"], where["size"]) == (int(r["gpu"]), int(r["start"]), int(r["size"])), trial
            assert sorted(int(u[1:]) for u in gone) == ks, trial


@pytest.mark.parametrize("policy", [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED])
@pytest.mark.parametrize("quirks", QUIRKS2)
@pytest.mark.parametrize("name", ["t16mix2", "t8tab"])
def test_node_score_fast_agrees_with_node_score_oracle(name, quirks, policy):
    """Unequal and empty nodes, whole occupancy bytes, ranges at unaligned bounds; FREEs of whole busy spans only, so that the dict side
    can name them as allocations."""
    rows = FIXTURES[name]()
    names = names_of(rows)
    srng = W.SplitMix64(300 + quirks + 2 * policy + len(name))
    rnd = random.Random(quirks + policy)
    placed = 0
    for trial in range(5):
        n_nodes = 1 + int(srng.next1() % 20)
        node_off = scoring_nodes(srng, n_nodes)
        G = int(node_off[-1])
        node_table = node_tables_for(rows, srng, n_nodes)
        occ = whole_bytes(srng, G)
        lo, hi = (0, G) if trial % 2 == 0 or G < 2 else sorted(rnd.sample(range(G + 1), 2))
        req = W.alloc_requests((srng.next(60) % np.uint64(len(names) + 1)).astype(np.uint8))
        req["profile"][req["profile"] == len(names)] = E.PROFILE_UNKNOWN
        req["op"][srng.next(60) % np.uint64(23) == 0] = E.OP_NOOP
        items = scoring_items(node_off, occ, rows, node_table)
        pods = []
        for i in range(len(req)):
            if srng.next1() % 8 == 0:                   # a FREE of a busy slice run, made an allocation of its own on the dict side
                g = int(srng.next1() % G)
                s = int(srng.next1() % 8)
                z = 1
                while s + z < 8 and int(occ[g]) >> (s + z) & 1 and srng.next1() % 2:
                    z += 1
                n = int(np.searchsorted(node_off, g, side="right")) - 1
                spec = items[n]["spec"]
                if all(int(occ[g]) >> x & 1 and ("p%d-%d" % (g, x)) in spec["prepared"] for x in range(s, s + z)):
                    for x in range(s, s + z):
                        del spec["prepared"]["p%d-%d" % (g, x)]
                    spec["allocations"]["old-%d" % i] = {"gpuUUID": "GPU-%07d" % g, "start": s, "size": z, "allocationStatus": "created"}
                    req[i] = (g, 0, E.OP_FREE, s, z)
                    pods.append({"op": "free", "uid": "old-%d" % i})
                    continue
            if req[i]["op"] == E.OP_ALLOC:
                p = int(req[i]["profile"])
                pods.append({"op": "alloc", "profile": names[p] if p < len(names) else "unknown", "uid": "pod-%d" % i})
            else:
                pods.append({"op": "noop"})
        out, after = NF.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
        got = NO.place_cr(items, pods, policy, quirks, lo, hi, names)
        for i in range(len(req)):
            if req[i]["op"] == E.OP_NOOP:
                assert int(out[i]["status"]) == E.ST_NOOP
                continue
            assert tuple(int(x) for x in out[i]) == NO.as_records([got[i]])[0], (trial, i, req[i])
        assert np.array_equal(after, NO.occupancy(items)), trial
        placed += int((out["status"] == E.ST_PLACED).sum())
    assert placed


@pytest.mark.parametrize("quirks", QUIRKS2)
def test_fast_place_gangs_agrees_with_ref_py_on_t8tab(quirks):
    """First-fit: the gang rules over ref_fast against reconcile_gated_pod on deep copies of the dicts, 8 tables, 16 names."""
    rows = t8tab()
    names = names_of(rows)
    rng = W.SplitMix64(800 + quirks)
    table_list = fixture_tables(rows)
    verdicts = set()
    for trial in range(4):
        n_nodes = 3 + int(rng.next1() % 10)
        node_off = np.concatenate([[0], np.cumsum(1 + (rng.next(n_nodes) % np.uint64(3)).astype(np.int64))]).astype(np.uint32)
        G = int(node_off[-1])
        node_table = t8tab_node_tables(rng, n_nodes)
        occ = whole_bytes(rng, G)
        n = 20 + int(rng.next1() % 40)
        prof = (rng.next(n) % np.uint64(16)).astype(np.uint8)
        req = W.alloc_requests(prof)
        off = [0]                                       # gangs of 1..5
        while off[-1] < n:
            off.append(min(n, off[-1] + 1 + int(rng.next1() % 5)))
        off = np.asarray(off, dtype=np.uint32)
        ref = oracle.Fast(node_off, rows, quirks, 0, node_table=node_table)
        ref.load(occ)
        got = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows, node_table))
        crs = GO.cluster_crs(node_off, node_table, occ, table_list)
        gangs = [[({"uid": "u%d" % i, "name": "p%d" % i}, names[prof[i]]) for i in range(a, b)] for a, b in zip(off[:-1], off[1:])]
        want = GO.ref_py_place_gangs(crs, gangs, quirks)
        for gi, ((a, b), (verdict, detail)) in enumerate(zip(zip(off[:-1], off[1:]), want)):
            recs = got[a:b]
            verdicts.add(verdict)
            if verdict == "placed":
                assert (recs["status"] == E.ST_PLACED).all(), (trial, gi)
                assert [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in recs] == \
                       [(int(x["gpuUUID"][4:]), x["start"], x["size"]) for x in detail], (trial, gi)
            else:
                assert recs["status"][detail] == E.ST_NO_CAPACITY, (trial, gi)
                assert (np.delete(recs["status"], detail) == E.ST_GANG_ABORTED).all(), (trial, gi)
        assert np.array_equal(ref.occupancy(), GO.cr_occupancy(crs)), trial
    assert verdicts == {"placed", "aborted"}


def test_candidate_masks_of_the_preempt_fixtures():
    """T16mix-2 under FIXED quirks places sizes 3, 5, 6 and 7; T16x8's rows all have a legal 8th start."""
    masks = {bin(candidate_mask(r["size"], s, E.QUIRKS_FIXED)).count("1") for r in t16mix(2) for s in r["starts"][:r["n_starts"]]}
    assert {3, 5, 6, 7, 8} <= masks
    assert all(candidate_mask(1, r["starts"][7], E.QUIRKS_REF_EXACT) for r in t16x8())
