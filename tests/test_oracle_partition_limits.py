"""The partitioned inventory at its limits, and the CPU pins of its checker (CPU only).

A partitioned inventory is one engine per rank, each owning a contiguous canonical GPU range [lo, hi); ``test_gpu_partition_limits.py``
runs every mechanism that joins the ranks (token ring, owner-gathered results, speculative ring, host-carried token) on the inputs built
here and compares each device byte with what this file derives:

  cut generators     ragged nodes of 1..9 GPUs and rank bounds for worlds 2..8 that cut through nodes and through one 4-byte occupancy
                     word, give a rank one GPU or exactly one node, make ranks very unequal, or sit on / off the speculative stage size
  rank_records       what EACH rank's own result array holds: the PLACED record on the rank that owns the GPU, the NO_CAPACITY default of
                     the whole inventory everywhere else, FREED / BAD_SPAN / BAD_PROFILE / NOOP identical on every rank
  trap_tables        node tables on which a rank-local default row would report another size than the whole inventory's
  ring_plan          the path islplace.cu's route / plan_pipeline / segment_geometry choose for a partitioned stream, per rank
  stream-id tags     the speculative rounds' record words carry 24 bits of the stream id: tests/spec_rounds_async_model.cpp shows what a
                     stale record with a matching tag does (the reason the engine speculates only under ids below 2^24)
"""
import math
import os
import subprocess

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W
from range_oracle import RangeFast
from test_oracle_inventory_limits import CHUNK, H100_SMS, MASK_BUDGET, SEG_MAX, SPEC_MAX_STAGES, SUB_MAX, SWEEP_BLOCK, max_segment_for
from test_oracle_table_limits import candidates, churn_batches, default_sizes, ragged_nodes, t8tab, t16x8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_STREAM_CHUNKS = 4096    # kMaxStreamChunks: chunks of one partitioned stream call
SPEC_RING_CHUNKS = 64       # kSpecRingChunks: chunks of one partitioned call that may speculate
SPEC_RING_IDS = 1 << 24     # kSpecRingIds: stream ids that may speculate
MAX_WORLD = 8               # isl_connect_spec_local / isl_ipc_connect_spec accept 2..8 ranks
CUT_KINDS = ("proportional", "word", "single", "node", "unequal", "sz", "off_sz")


# ---- cut generators --------------------------------------------------------------------------------------------------------------------
def ragged(rng, n_nodes):
    """Node offsets of n_nodes nodes of 1..9 GPUs each."""
    return ragged_nodes(rng, n_nodes, max_gpus=9)


def stage_size(G):
    """sz of plan_pipeline's ring branch: the power-of-two stage size (>= 64) that keeps the whole sequence within kSpecMaxStages."""
    sz = 64
    while -(-G // sz) > SPEC_MAX_STAGES:
        sz *= 2
    return sz


def cuts(kind, node_off, world, rng):
    """world + 1 ascending bounds over G = node_off[-1] GPUs, every rank non-empty, of the given kind."""
    node_off = np.asarray(node_off, dtype=np.int64)
    G = int(node_off[-1])
    inner = set(int(b) for b in node_off[1:-1])
    r = lambda n: int(rng.next1() % np.uint64(n))
    if kind == "proportional":          # dist.partition_bounds below world x 512 GPUs: wherever G * r // world lands
        assert G < world * 512
        b = [G * k // world for k in range(world)] + [G]
    elif kind == "word":                # interior cuts inside a node and inside a 4-byte occupancy word
        b = [0]
        for k in range(1, world):
            x = G * k // world
            while x % 4 == 0 or x in inner or x <= b[-1]:
                x += 1
            b.append(x)
        b.append(G)
    elif kind in ("single", "node"):    # rank 1 holds one GPU inside a node, or exactly one whole node
        n = len(node_off) - 1
        if kind == "single":
            i = next(i for i in range(n // 3, n) if node_off[i + 1] - node_off[i] >= 3)
            a = int(node_off[i]) + 1
            b1 = [a, a + 1]
        else:
            i = next(i for i in range(n // 3, n) if node_off[i + 1] - node_off[i] >= 4)
            b1 = [int(node_off[i]), int(node_off[i + 1])]
        if world == 2:                  # the last rank: one GPU, or the last node
            b = [0, G - 1, G] if kind == "single" else [0, int(node_off[-2]), G]
        else:
            rest = np.linspace(b1[1], G, world - 1)[1:-1].astype(np.int64).tolist()
            b = [0] + b1 + [int(x) for x in rest] + [G]
    elif kind == "unequal":             # widths from one GPU to most of the inventory
        w = [1 + r(3)] + [3 + r(40) for _ in range(world - 2)]
        b = [0] + np.cumsum(w).tolist()
        b.append(G)
    elif kind in ("sz", "off_sz"):      # multiples of the stage size, very unequal; off_sz moves one interior cut off it
        sz = stage_size(G)
        units = G // sz
        w = [1] + [1 + r(2) for _ in range(world - 2)]
        b = [0] + (np.cumsum(w) * sz).tolist()
        assert b[-1] < units * sz
        b.append(G)
        if kind == "off_sz":
            k = 1 + r(world - 1)
            b[k] += 1 + r(sz - 1)
            assert b[k] < b[k + 1]
    else:
        raise ValueError(kind)
    b = [int(x) for x in b]
    assert len(b) == world + 1 and b[0] == 0 and b[-1] == G and all(x < y for x, y in zip(b, b[1:])), (kind, b)
    return b


def inventory(seed, world, kind, n_nodes=700):
    """(node_off, occ, bounds) of one case: ragged nodes, ~1/4 busy slices, the cuts of the kind."""
    rng = W.SplitMix64(seed)
    if kind == "proportional":                  # G < world x 512, and at least one cut inside a node
        n_nodes = min(n_nodes, world * 80)
        while True:
            node_off = ragged(rng, n_nodes)
            G = int(node_off[-1])
            if any(G * k // world not in set(node_off.tolist()) for k in range(1, world)):
                break
    else:
        node_off = ragged(rng, n_nodes)
    G = int(node_off[-1])
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    return node_off, occ, cuts(kind, node_off, world, rng)


def edges(node_off, b):
    """The edges a bounds list reaches."""
    node_off = np.asarray(node_off, dtype=np.int64)
    G = int(node_off[-1])
    nodes = set(int(x) for x in node_off)
    w = np.diff(b)
    sz = stage_size(G)
    one_node = any(b[k] in nodes and b[k + 1] in nodes and np.searchsorted(node_off, b[k], side="right") == np.searchsorted(node_off, b[k + 1], side="left")
                   for k in range(len(b) - 1))
    return {
        "through_node": any(x not in nodes for x in b[1:-1]),
        "through_word": any(x % 4 != 0 and x not in nodes for x in b[1:-1]),
        "one_gpu": bool((w == 1).any()),
        "one_node": one_node,
        "unequal": int(w.max()) >= 8 * int(w.min()),
        "on_sz": all(x % sz == 0 for x in b[:-1]),
        "off_sz": sum(x % sz != 0 for x in b[1:-1]) == 1,
    }


WANT_EDGE = {"proportional": "through_node", "word": "through_word", "single": "one_gpu", "node": "one_node", "unequal": "unequal",
             "sz": "on_sz", "off_sz": "off_sz"}


@pytest.mark.parametrize("world", range(2, MAX_WORLD + 1))
@pytest.mark.parametrize("kind", CUT_KINDS)
def test_every_cut_generator_reaches_its_edge(kind, world):
    for seed in range(3):
        node_off, _, b = inventory(100 * world + seed, world, kind)
        e = edges(node_off, b)
        assert e[WANT_EDGE[kind]], (kind, world, b, e)
        if kind == "word":
            assert e["through_node"] and any(x % 4 in (1, 2, 3) for x in b[1:-1])
        if kind in ("sz", "off_sz"):
            assert e["unequal"] or world == 2
            assert int(node_off[-1]) <= 64 * 64 and stage_size(int(node_off[-1])) == 64     # G <= 4096: stages fit half an H100


def test_cut_kinds_cover_every_edge_together():
    seen = set()
    for world in range(2, MAX_WORLD + 1):
        for kind in CUT_KINDS:
            node_off, _, b = inventory(7 * world, world, kind)
            seen |= {k for k, v in edges(node_off, b).items() if v}
    assert seen == set(WANT_EDGE.values())
    assert {int(x) for x in np.diff(ragged(W.SplitMix64(3), 400))} == set(range(1, 10))


# ---- per-rank expected records -------------------------------------------------------------------------------------------------------
def rank_records(req, res, lo, hi, dflt):
    """Rank [lo, hi)'s own result array, from the whole inventory's records ``res``: a PLACED record stays on the rank that owns its GPU;
    on every other rank that ALLOC reports NO_CAPACITY with the whole inventory's default size.  Every other record is the same on all
    ranks."""
    out = res.copy()
    away = (res["status"] == E.ST_PLACED) & ((res["gpu"] < lo) | (res["gpu"] >= hi))
    out["gpu"][away], out["start"][away], out["status"][away] = E.GPU_NONE, E.START_NONE, E.ST_NO_CAPACITY
    out["size"][away] = np.asarray(dflt, dtype=np.uint8)[req["profile"][away]]
    return out


def rank_occupancy(occ_before, occ_after, lo, hi):
    """A rank's whole occupancy after a call: the oracle's bytes inside [lo, hi), the loaded bytes everywhere else."""
    out = np.array(occ_before, dtype=np.uint8)
    out[lo:hi] = occ_after[lo:hi]
    return out


def dflt_of(rows, node_off, node_table):
    if rows.ndim == 1:
        return [int(s) for s in rows["size"]] + [0] * (E.MAX_PROFILES - len(rows))
    d = default_sizes(rows, node_table)
    return d + [0] * (E.MAX_PROFILES - len(d))


def ring_requests(rng, ref, sizes, n_names, G):
    """churn_batches plus malformed FREEs (gpu >= G, start + size > 8), a NOOP and a FREE of slice 7 anywhere in every batch of >= 4."""
    out = []
    for req, _ in churn_batches(rng, oracle.Fast(ref.node_off, ref.rows, ref.quirks, node_table=ref.node_table), sizes, n_names):
        req = req.copy()
        if len(req) >= 4:
            k = np.argsort(rng.next(len(req)), kind="stable")[:4]
            req[k[0]] = (G + int(k[0]) % 5, 0, E.OP_FREE, 0, 1)
            req[k[1]] = (int(k[1]) % G, 0, E.OP_FREE, 5, 4)
            req["op"][k[2]] = E.OP_NOOP
            req[k[3]] = (int(rng.next1() % np.uint64(G)), 0, E.OP_FREE, 7, 1)      # well-formed: FREED, applied by its rank only
        out.append(req)
    return out


class _Ref:
    """oracle.Fast with what ring_requests needs to rebuild it."""
    def __init__(self, node_off, rows, quirks, node_table, occ):
        self.node_off, self.rows, self.quirks, self.node_table = node_off, rows, quirks, node_table
        self.fast = oracle.Fast(node_off, rows, quirks, node_table=node_table)
        self.fast.load(occ)


def sequential_ring(node_off, rows, occ, bounds, batches, quirks, node_table):
    """The ring restated with range_oracle alone: rank after rank, each a RangeFast over its range that sees every request the ranks in
    front did not place (those turn into NOOPs).  Returns per batch the list of per-rank records and the positions handed over."""
    ranks = [RangeFast(node_off, rows, occ, lo, hi, quirks, node_table=node_table) for lo, hi in zip(bounds, bounds[1:])]
    out = []
    for req in batches:
        taken = np.zeros(len(req), dtype=bool)
        per_rank = []
        for rf in ranks:
            sub = req.copy()
            sub["op"][taken] = E.OP_NOOP
            res = rf.place(sub)
            per_rank.append((res, taken.copy()))
            taken |= (req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)
        out.append(per_rank)
    return out, ranks


@pytest.mark.parametrize("world", [2, 3, 5, 8])
@pytest.mark.parametrize("kind", ["word", "single", "node", "unequal"])
def test_rank_records_agree_with_range_oracle_and_merge_to_fast(kind, world):
    rng = W.SplitMix64(5000 + world)
    node_off = ragged(rng, 30 + 4 * world)
    G = int(node_off[-1])
    b = cuts(kind, node_off, world, rng)
    tabled = world % 2 == 1
    rows = t8tab() if tabled else E.make_profiles(tables.H100_80GB)
    node_table = trap_tables(rng, node_off, b) if tabled else None
    quirks = E.QUIRKS_FIXED if tabled else E.QUIRKS_REF_EXACT
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    ref = _Ref(node_off, rows, quirks, node_table, occ)
    batches = ring_requests(rng, ref, [40, 0, 90, 7], rows.shape[-1], G)
    dflt = dflt_of(rows, node_off, node_table)
    seq, ranks = sequential_ring(node_off, rows, occ, b, batches, quirks, node_table)
    for req, per_rank in zip(batches, seq):
        want = ref.fast.place(req)
        mine = [rank_records(req, want, lo, hi, dflt) for lo, hi in zip(b, b[1:])]
        for (res, taken), m in zip(per_rank, mine):
            assert np.array_equal(res[~taken], m[~taken])
            assert (m["status"][taken] == E.ST_NO_CAPACITY).all()
        merged = np.minimum.reduce([m.view(np.int64) for m in mine]).view(E.RESULT_DTYPE)
        assert np.array_equal(merged, want)
        if len(req) >= 4:
            st = want["status"]
            assert {E.ST_FREED, E.ST_BAD_SPAN, E.ST_NOOP} <= set(st.tolist())
    final = ref.fast.occupancy()
    for rf, lo, hi in zip(ranks, b, b[1:]):
        assert np.array_equal(rf.occupancy(), rank_occupancy(occ, final, lo, hi))


def test_merge_hides_a_rank_local_default_and_freed_for_bad_span():
    """Why each rank's array is compared, not only the merge: a rank that reported its own node's default size, or FREED for a malformed
    FREE, disappears in the element-wise MIN whenever its value is the smaller one."""
    rec = np.zeros(2, dtype=E.RESULT_DTYPE)
    rec[0] = (E.GPU_NONE, E.START_NONE, 4, E.ST_NO_CAPACITY)
    rec[1] = (5000, 5, 4, E.ST_BAD_SPAN)
    wrong = rec.copy()
    wrong["size"][0] = 2                                  # a rank-local default row of 2 slices
    wrong["status"][1] = E.ST_FREED
    merged = np.minimum(rec.view(np.int64), wrong.view(np.int64)).view(E.RESULT_DTYPE)
    assert np.array_equal(merged, wrong) and not np.array_equal(merged, rec)


# ---- node tables where the default row matters ----------------------------------------------------------------------------------------
TRAP_NAME = 15      # t8tab: profile 15 is known to table 7 only


def trap_tables(rng, node_off, bounds):
    """Table of every node for t8tab rows: tables 0..6 at random, table 7 (the only one that knows profile 15) only on nodes that begin in
    the last rank, node 0 on table 2 (which does not know every name)."""
    n = len(node_off) - 1
    node_table = (rng.next(n) % np.uint64(7)).astype(np.uint8)
    node_table[0] = 2
    first = np.asarray(node_off[:-1], dtype=np.int64)
    last_rank = np.flatnonzero(first >= bounds[-2])
    node_table[last_rank[:: 2]] = 7
    return node_table


def local_default(rows, node_off, node_table, lo, hi, p):
    """What a rank would report if it took the default row from the first node of ITS range whose table has the name (0: none)."""
    node_off = np.asarray(node_off, dtype=np.int64)
    for i in range(len(node_off) - 1):
        if node_off[i + 1] > lo and node_off[i] < hi and rows["n_starts"][node_table[i], p]:
            return int(rows["size"][node_table[i], p])
    return 0


@pytest.mark.parametrize("world", range(3, MAX_WORLD + 1))
def test_trap_tables_make_a_rank_local_default_wrong(world):
    rows = t8tab()
    node_off, _, b = inventory(900 + world, world, "word")
    node_table = trap_tables(W.SplitMix64(world), node_off, b)
    dflt = default_sizes(rows, node_table)
    first15 = next(i for i, t in enumerate(node_table) if rows["n_starts"][t, TRAP_NAME])
    rank_of = lambda g: int(np.searchsorted(b, g, side="right")) - 1
    assert rank_of(int(node_off[first15])) >= 2                         # the first node that knows the name lies in rank 2 or later
    assert dflt[TRAP_NAME] == int(rows["size"][7, TRAP_NAME]) > 0
    assert local_default(rows, node_off, node_table, b[0], b[1], TRAP_NAME) == 0     # rank 0 has no node with the name at all
    # a name whose size differs between the tables, and a rank whose local default differs from the whole inventory's
    known = rows["n_starts"] > 0
    assert any(len({int(rows["size"][t, p]) for t in range(8) if known[t, p]}) > 1 for p in range(16))
    wrong = [(r, p) for r in range(world) for p in range(16)
             if local_default(rows, node_off, node_table, b[r], b[r + 1], p) != dflt[p]]
    assert [1 for r, p in wrong if p != TRAP_NAME], wrong                # not only the trap name


# ---- the ring's plan, restated ---------------------------------------------------------------------------------------------------------
def ring_plan(G, bounds, sizes, n_cand, sms=H100_SMS, max_gpus=None, spec_world=0, ring_world=0, mode="auto", window=0, stream_id=1):
    """islplace.cu route / plan_pipeline / segment_geometry for isl_place_stream_partitioned on every rank: ("erange", None), or
    ("spec" | "plain", [n_seg of every rank]).  spec_world: ranks wired with isl_connect_spec_local (0: none); ring_world:
    isl_set_ring_world; mode: isl_set_speculation; window: isl_set_causal_window (it applies on a ring only with ring_world set)."""
    ceil = lambda a, c: -(-a // c)
    max_gpus = max_gpus or G
    n_chunks = sum(ceil(n, CHUNK) for n in sizes)
    if n_chunks > MAX_STREAM_CHUNKS:
        return ("erange", None)
    if len(sizes) * ceil(max_gpus, SWEEP_BLOCK) * SWEEP_BLOCK > MASK_BUDGET:
        return ("erange", None)
    window = window if ring_world else 0
    auto_spec = len(sizes) == 1 or 1 <= window <= 3
    seg_cap = max_segment_for(n_cand)
    widths = [hi - lo for lo, hi in zip(bounds, bounds[1:])]
    if stream_id < SPEC_RING_IDS and spec_world >= 2 and (mode == "on" or (mode == "auto" and auto_spec)):
        sz = stage_size(G)
        ok = (sz <= SEG_MAX and spec_world == ring_world and n_chunks <= SPEC_RING_CHUNKS and bounds[-1] == G and
              all(x % sz == 0 or x == G for x in bounds) and all(w > 0 and ceil(w, sz) <= sms for w in widths))
        if ok and sz <= seg_cap:
            return ("spec", [ceil(w, sz) for w in widths])
    avg = sum(sizes) / n_chunks
    target = int(min(sms, max(1.0, math.floor(math.sqrt(max(1.0, n_chunks - 1.0) * min(avg, 3.5 * G) * (0.0326 / 1.57)) + 0.5))))
    if seg_cap < 64:
        return ("erange", None)
    sub = min(seg_cap, max(64, (ceil(G, target) + 63) // 64 * 64))
    target = max(target, min(sms, ceil(ceil(G, sub), SUB_MAX)))
    n_sub = max(1, ceil(ceil(G, sub), target))
    if n_sub > SUB_MAX:
        return ("erange", None)
    n_seg = [max(1, ceil(w, sub * n_sub)) for w in widths]
    return ("erange", None) if max(n_seg) > sms else ("plain", n_seg)


def total_ctas(plan):
    """Co-resident k_pipeline CTAs over all ranks (device buffers: no copier CTA)."""
    return sum(plan[1])


def test_ring_plan_speculates_only_where_the_engine_may():
    n_cand = len(candidates(t16x8(), E.QUIRKS_REF_EXACT))
    G = 4000
    on = [0, 64, 192, 1024, 2048, G]
    kw = dict(spec_world=5, ring_world=5, mode="on")
    p = ring_plan(G, on, [5000], n_cand, **kw)
    assert p[0] == "spec" and p[1] == [1, 2, 13, 16, 31] and total_ctas(p) == 63 <= H100_SMS // 2
    off = list(on)
    off[2] += 1
    assert ring_plan(G, off, [5000], n_cand, **kw)[0] == "plain"                          # one bound off the stage size
    assert ring_plan(G, on, [300] * 64, n_cand, **kw)[0] == "spec"                        # 64 chunks
    assert ring_plan(G, on, [300] * 65, n_cand, **kw)[0] == "plain"                       # 65 chunks
    assert ring_plan(G, on, [5000], n_cand, spec_world=5, ring_world=4, mode="on")[0] == "plain"
    assert ring_plan(G, on, [5000], n_cand, spec_world=5, ring_world=5)[0] == "spec"      # auto: one batch
    assert ring_plan(G, on, [50, 50], n_cand, spec_world=5, ring_world=5)[0] == "plain"   # auto: two batches, no window
    assert ring_plan(G, on, [50, 50], n_cand, spec_world=5, ring_world=5, window=2)[0] == "spec"
    for sid in (1, 32767, 32768, SPEC_RING_IDS - 1):
        assert ring_plan(G, on, [5000], n_cand, stream_id=sid, **kw)[0] == "spec"
    for sid in (SPEC_RING_IDS, SPEC_RING_IDS + 1, 2 ** 32 - 1):
        assert ring_plan(G, on, [5000], n_cand, stream_id=sid, **kw)[0] == "plain"
    # the refusals
    assert ring_plan(G, on, [1] * 4095 + [CHUNK + 1], n_cand) == ("erange", None)       # 4 097 chunks
    assert ring_plan(G, on, [1] * 4094 + [CHUNK + 1], n_cand)[0] == "plain"              # 4 096
    assert ring_plan(G, on, [10] * 17, n_cand, max_gpus=1 << 24) == ("erange", None)      # 17 x 16 MiB of free masks
    assert ring_plan(G, on, [10] * 16, n_cand, max_gpus=1 << 24)[0] == "plain"
    # a 65 536-GPU, 128-stage sequence is config 4's 8-GPU geometry, beyond half of one H100
    big = [65536 * k // 8 for k in range(8)] + [65536]
    assert total_ctas(ring_plan(65536, big, [5000], n_cand, spec_world=8, ring_world=8, mode="on")) == 128 > H100_SMS // 2


@pytest.mark.parametrize("world", range(2, MAX_WORLD + 1))
@pytest.mark.parametrize("kind", CUT_KINDS)
def test_every_gpu_case_fits_half_an_h100(kind, world):
    node_off, _, b = inventory(100 * world, world, kind)
    G = int(node_off[-1])
    for rows, q in ((t16x8(), E.QUIRKS_REF_EXACT), (t8tab(), E.QUIRKS_FIXED)):
        n_cand = len(candidates(rows, q))
        for sizes in ([70_000, 0, 3000], [300] * 64, [300] * 65, [5000]):
            for kw in ({}, dict(spec_world=world, ring_world=world, mode="on")):
                p = ring_plan(G, b, sizes, n_cand, **kw)
                assert p[0] != "erange" and total_ctas(p) <= H100_SMS // 2, (kind, world, sizes, kw, p)
                if kw and kind == "sz" and len(sizes) <= 64:
                    assert p[0] == "spec"
                if kind == "off_sz" or len(sizes) == 65 or not kw:
                    assert p[0] == "plain"


# ---- stream-id tags of the speculative rounds -------------------------------------------------------------------------------------------
def record_tag(stream_id, rnd):
    """The upper word of a round record (isl_kernels.cuh resolve_rounds / exchange_round): 24 bits of the id, then the round."""
    return ((stream_id & 0xFFFFFF) << 8) | rnd


def final_tag(stream_id):
    return ((stream_id & 0xFFFFFF) << 8) | 0xFF


def test_record_tags_repeat_every_2_24_ids_and_cleared_memory_matches_only_round_0_of_tag_0():
    for s in (1, 12345, SPEC_RING_IDS - 1):
        assert record_tag(s, 3) == record_tag(s + SPEC_RING_IDS, 3) and final_tag(s) == final_tag(s + SPEC_RING_IDS)
    # distinct ids below 2^24 never share a tag, and none of them is 0
    assert len({record_tag(s, 0) for s in range(1, 1 << 16)}) == (1 << 16) - 1 and record_tag(1, 0) != 0
    # ids with low 24 bits 0 (2^24, 2^25, ...): the round-0 mass words match a cleared word; rounds 1.. and the final words never do
    assert record_tag(SPEC_RING_IDS, 0) == 0
    assert all(record_tag(SPEC_RING_IDS, r) != 0 for r in range(1, 160)) and final_tag(SPEC_RING_IDS) != 0


def _async_model(tmp_path):
    exe = str(tmp_path / "spec_rounds_async_model")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "spec_rounds_async_model.cpp")], check=True)
    return exe


def test_a_stale_record_with_the_current_tag_changes_a_decision(tmp_path):
    """Stream ids s and s + 2^24 share every record tag, and the ring's shared record memory keeps the earlier call's words: a stage
    then takes the earlier call's exit heads or final record as current and certifies a wrong entry.  Hence only ids below 2^24
    speculate on the ring."""
    out = subprocess.run([_async_model(tmp_path), "600", "0", "1"], capture_output=True, text=True)
    assert out.returncode != 0 and "unsound certification" in out.stdout, out.stdout[-2000:]


def test_a_zero_tag_on_cleared_memory_only_moves_predictions(tmp_path):
    """With the low 24 bits of the tag 0 only the round-0 mass words match cleared memory: a stage may predict from masses of 0, and the
    rounds still certify only true entries."""
    out = subprocess.run([_async_model(tmp_path), "2000", "0", "2"], capture_output=True, text=True)
    assert out.returncode == 0 and "ok (2000 cases)" in out.stdout, out.stdout[-2000:]
