"""Every gang kind under node scoring (isl_place_gangs on an engine created with ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_NODE_SCORE_ALL)
on the H100: the node-scored k_ganglocal instantiations of few-node, elastic and balanced gangs against the brute force of
tests/gang_score_all_fast.cpp (records, occupancy, stats.placed) on random calls, the known-answer vectors, 2^20 GPUs, 2^20 one-GPU
nodes, every edge of the CTA layout and the table limits; C7, C4 (a), C4 (c), C6 (c) and M5 (b) device against device; C1-C2 and the
codes of every engine state; the reconciler and the C++ mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_score_all_fast as GSA
import gang_score_all_oracle as GSAO
from test_gpu_gang_few import cr_cluster, device, pods, random_call
from test_oracle_gang_topology_limits import CASES, FIXTURES, LAYOUT_CASES, case_ids, gang_plan, layout_cases, small_gangs
from test_oracle_request_major_limits import gang_call, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]
SCORE = E.FLAG_GANG_NODE_SCORE
ALL = E.FLAG_GANG_NODE_SCORE | E.FLAG_GANG_NODE_SCORE_ALL
PER_GANG = E.FLAG_GANG_LOCALITY | E.FLAG_GANG_BALANCED
# (engine flags besides ALL, the brute force's locality): each gang's byte, or the engine's locality for every gang
MODES = {"per_gang": (PER_GANG, GSA.PER_GANG), "locality": (E.FLAG_GANG_LOCALITY, GSA.PER_GANG), "few": (E.FLAG_GANG_FEW_NODES, 2),
         "one": (E.FLAG_GANG_ONE_NODE, 1), "distinct": (E.FLAG_GANG_DISTINCT_NODES, 3), "any": (0, 0)}
# the new and changed instantiations: <per_gang, [min,] node_score, balanced>, <per_gang, min, node_score>, <few_nodes, node_score>
# and <per_gang, node_score> with few-node bytes
KERNELS = [("per_gang", False), ("per_gang", True), ("locality", True), ("few", False), ("few", True), ("one", True),
           ("distinct", True), ("any", True), ("locality", False)]


def engine(node_off, rows, occ, policy, flags, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16):
    eng = E.Engine(max_gpus=max(4097, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if np.asarray(rows).ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def bytes_for(rng, n_gangs, mode):
    """Locality bytes: every byte 0..7 and 255 on a balanced engine, 0..3 on a locality engine."""
    b = (rng.next(n_gangs) % np.uint64(8 if mode == "per_gang" else 4)).astype(np.int64)
    if mode == "per_gang":
        b[rng.next(n_gangs) % np.uint64(11) == 0] = 255
    return b


def with_bytes(req, off, rng, mode, elastic):
    req = req.copy()
    alloc = req["op"] == E.OP_ALLOC
    sizes = np.diff(off.astype(np.int64))
    if MODES[mode][1] is GSA.PER_GANG:
        req["start"][alloc] = np.repeat(bytes_for(rng, len(off) - 1, mode), sizes)[alloc]
    if elastic:
        req["size"][alloc] = np.repeat((rng.next(len(off) - 1) % np.uint64(6)).astype(np.int64), sizes)[alloc]
    return req


def check(node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, mode, elastic, what=""):
    """One call on an engine with the bit against the brute force: records, occupancy and stats.placed."""
    flags, loc = MODES[mode]
    eng = engine(node_off, rows, occ, policy, ALL | flags | (E.FLAG_GANG_MIN_MEMBERS if elastic else 0), quirks, node_table,
                 max_batch=max(16, len(req)))
    if (lo, hi) != (0, int(node_off[-1])):
        eng.set_partition(lo, hi)
    want, occ_want, placed = GSA.place_gangs(node_off, rows, occ, req, off, policy, loc, quirks, node_table, lo, hi, elastic)
    eng.reset_stats()
    got = eng.place_gangs(req, off)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    assert eng.stats()["placed"] == placed, what
    eng.close()
    return got


@pytest.mark.parametrize("vector", GSAO.kat_vectors(), ids=lambda v: v["name"])
def test_kat(vector):
    x = GSAO.vector_inputs(vector)
    mode = "per_gang" if x["locality"] is None else {1: "one", 2: "few", 3: "distinct", 0: "any"}[x["locality"]]
    got = check(x["node_off"], x["rows"], x["node_table"], x["occ"], x["requests"], x["gang_off"], x["quirks"], x["policy"], x["lo"],
                x["hi"], mode, x["elastic"], vector["name"])
    assert [tuple(int(v) for v in r) for r in got] == GSAO.expected(vector)[0]


@pytest.mark.parametrize("mode,elastic", KERNELS)
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_vs_brute_force(policy, quirks, mode, elastic):
    """Small random clusters: one or three node tables, partitions that cut nodes, FREEs, NOOPs and unknown profiles."""
    rng = SplitMix64(12100 + 100 * policy + 10 * quirks + KERNELS.index((mode, elastic)))
    for i in range(30):
        n_nodes = 1 + int(rng.next1() % 12)
        node_off = np.cumsum([0] + [int(rng.next1() % 5) + (k == 0) for k in range(n_nodes)]).astype(np.uint32)
        G = int(node_off[-1])
        if i % 2:
            _, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
            node_table = (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8)
        else:
            rows, node_table = E.make_profiles(tables.H100_80GB), None
        occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
        req, off = random_call(rng, G, np.asarray(rows).shape[-1], 1 + int(rng.next1() % 30), 8)
        req = with_bytes(req, off, rng, mode, elastic)
        lo, hi = (0, G) if i % 3 else sorted((int(rng.next1() % G), 1 + int(rng.next1() % G)))
        if lo >= hi:
            lo, hi = 0, G
        check(node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, mode, elastic, i)


@pytest.mark.parametrize("mode,elastic", KERNELS)
@pytest.mark.parametrize("policy", POLICIES)
def test_large_vs_brute_force(policy, mode, elastic):
    """Thousands of GPUs in nodes of 1-16 with three node tables: many CTAs, gangs of up to 8, a partition that cuts nodes."""
    rng = SplitMix64(12200 + 10 * policy + KERNELS.index((mode, elastic)))
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 16) for _ in range(700)]).astype(np.uint32)
    G = int(node_off[-1])
    _, rows = E.make_profile_tables([tables.H100_80GB, tables.A30_24GB, tables.A100_40GB])
    node_table = (rng.next(700) % np.uint64(3)).astype(np.uint8)
    occ = (rng.next(G) & np.uint64(0x7B)).astype(np.uint8)
    req, off = random_call(rng, G, rows.shape[1], 1500, 8)
    req = with_bytes(req, off, rng, mode, elastic)
    for part in ((0, G), (int(rng.next1() % 100) + 3, G - 50)):
        check(node_off, rows, node_table, occ, req, off, E.QUIRKS_FIXED, policy, *part, mode, elastic, part)


@pytest.mark.parametrize("mode,elastic", [("per_gang", True), ("few", False), ("locality", True)])
@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy, mode, elastic):
    """A 2^20-GPU partition of 8-GPU nodes (the cap), and 2^20 one-GPU nodes (node scoring's node cap)."""
    rng = SplitMix64(12300 + 10 * policy + len(mode) + elastic)
    rows = E.make_profiles(tables.H100_80GB)
    for node_off in (np.arange(0, (1 << 20) + 1, 8, dtype=np.uint32), np.arange((1 << 20) + 1, dtype=np.uint32)):
        G = int(node_off[-1])
        occ = whole_bytes(rng, G, dense=True)
        req, off = random_call(rng, G, len(rows), 120, 6)
        req = with_bytes(req, off, rng, mode, elastic)
        got = check(node_off, rows, None, occ, req, off, E.QUIRKS_REF_EXACT, policy, 0, G, mode, elastic, len(node_off))
        assert (got["status"] == E.ST_PLACED).any()


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_edges(case):
    """Every edge of the CTA layout built from this device's SM count and the balanced instantiation's shared-memory opt-in (its 256 B of
    static shared memory), shares on both sides of the shared / global memory switch among them, 8 node tables of widths 4-8."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    assert edge(gang_plan(node_off, lo, hi, sms, optin - 256)), case
    i = LAYOUT_CASES.index(case)
    rng = SplitMix64(12400 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    off = small_gangs(rng, 300, 8)
    req = with_bytes(gang_call(rng, G, 16, 300), off, rng, "per_gang", True)
    check(node_off, t8tab(), node_table, whole_bytes(rng, G, dense=True), req, off, E.QUIRKS_FIXED, POLICIES[i % 2], lo, hi, "per_gang",
          True, case)


@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_table_limits(name, quirks):
    """16 profiles and 8 node tables: every fixture of the table-limit suite, balanced and elastic per-gang bytes and few-node gangs."""
    rows = FIXTURES[name]()
    rng = SplitMix64(12500 + CASES.index((name, quirks)))
    n_nodes = 300
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 8) for _ in range(n_nodes)]).astype(np.uint32)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes) if np.asarray(rows).ndim == 2 else None
    n_names = np.asarray(rows).shape[-1]
    for k, (mode, elastic) in enumerate((("per_gang", True), ("few", False))):
        off = small_gangs(rng, 600, 6)
        req = with_bytes(gang_call(rng, G, n_names, 600), off, rng, mode, elastic)
        check(node_off, rows, node_table, whole_bytes(rng, G), req, off, quirks, POLICIES[k], 0, G, mode, elastic, (name, mode))


def run(eng, req, off):
    eng.reset_stats()
    return eng.place_gangs(req, off), eng.read_occupancy(), eng.stats()["placed"]


@pytest.mark.parametrize("policy", POLICIES)
def test_c7_bit_changes_nothing_for_bytes_0_1_3(policy):
    """C7, device against device: bytes 0, 1 and 3 without MIN return what the engine without the bit returns."""
    rng = SplitMix64(12600 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 12) for _ in range(400)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 2000, 6)
    alloc = req["op"] == E.OP_ALLOC
    req["start"][alloc] = np.repeat(np.array([0, 1, 3])[(rng.next(len(off) - 1) % np.uint64(3)).astype(np.int64)],
                                    np.diff(off.astype(np.int64)))[alloc]
    for extra in (E.FLAG_GANG_LOCALITY, E.FLAG_GANG_LOCALITY | E.FLAG_GANG_BALANCED):
        a = engine(node_off, rows, occ, policy, ALL | extra)
        b = engine(node_off, rows, occ, policy, SCORE | E.FLAG_GANG_LOCALITY)
        ra, rb = run(a, req, off), run(b, req, off)
        assert np.array_equal(ra[0], rb[0]) and np.array_equal(ra[1], rb[1]) and ra[2] == rb[2], extra
        a.close()
        b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_c4a_whole_few_node_gang_is_one_node(policy):
    """C4 (a), device against device: a few-node gang that some node takes whole gets the records and occupancy of the one-node scored
    engine (N5)."""
    rng = SplitMix64(12700 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 4) for _ in range(200)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
    few = engine(node_off, rows, occ, policy, ALL | E.FLAG_GANG_FEW_NODES)
    one = engine(node_off, rows, occ, policy, SCORE | E.FLAG_GANG_ONE_NODE)
    seen = 0
    for _ in range(40):
        req = alloc_requests((rng.next(1 + int(rng.next1() % 8)) % np.uint64(len(rows))).astype(np.uint8))
        off = [0, len(req)]
        b = run(one, req, off)
        if b[2] == len(req):
            a = run(few, req, off)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]
            seen += 1
        else:
            few.load_inventory(node_off, b[1])               # keep both engines on one occupancy
    assert seen > 10
    few.close()
    one.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_c4c_c6c_one_node_equals_first_fit_engine(policy):
    """C4 (c) and C6 (c), device against device: a partition inside one node, and a one-node inventory, equal a FIRST_FIT engine with the
    same gang flags (records and occupancy)."""
    rng = SplitMix64(12800 + policy)
    rows = E.make_profiles(tables.A100_40GB)
    for flags, mode in ((E.FLAG_GANG_FEW_NODES, "few"), (E.FLAG_GANG_FEW_NODES | E.FLAG_GANG_MIN_MEMBERS, "few"),
                        (PER_GANG, "per_gang"), (PER_GANG | E.FLAG_GANG_MIN_MEMBERS, "per_gang")):
        for node_off, part in ((node_offsets(8, 64), (70, 120)), (np.array([0, 300], dtype=np.uint32), None)):
            G = int(node_off[-1])
            occ = (rng.next(G) & np.uint64(0x5D)).astype(np.uint8)
            req, off = random_call(rng, G, len(rows), 300, 5)
            req = with_bytes(req, off, rng, mode, bool(flags & E.FLAG_GANG_MIN_MEMBERS))
            a, b = engine(node_off, rows, occ, policy, ALL | flags), engine(node_off, rows, occ, E.POLICY_FIRST_FIT, flags)
            if part:
                a.set_partition(*part)
                b.set_partition(*part)
            assert np.array_equal(a.place_gangs(req, off), b.place_gangs(req, off)), flags
            assert np.array_equal(a.read_occupancy(), b.read_occupancy()), flags
            a.close()
            b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_m5b_trimmed_gang_equals_cut_gang(policy):
    """M5 (b) under C5, device against device: a gang trimmed at f gets the records and occupancy of its first f members placed on the
    engine without MIN, where they commit; every locality byte."""
    rng = SplitMix64(12900 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 3) for _ in range(60)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
    el = engine(node_off, rows, occ, policy, ALL | PER_GANG | E.FLAG_GANG_MIN_MEMBERS)
    cut = engine(node_off, rows, occ, policy, ALL | PER_GANG)
    trims = 0
    for i in range(200):
        req = alloc_requests((rng.next(4 + int(rng.next1() % 12)) % np.uint64(len(rows))).astype(np.uint8))
        req["start"] = [0, 1, 2, 3, 4, 5, 255][i % 7]
        req["size"] = 1 + int(rng.next1() % 3)
        before = el.read_occupancy()
        got, after, placed = run(el, req, [0, len(req)])
        if not 0 < placed < len(req):
            cut.load_inventory(node_off, after)
            continue
        c = req[:placed].copy()
        c["size"] = 0
        cut.load_inventory(node_off, before)
        want = run(cut, c, [0, placed])
        assert want[2] == placed and np.array_equal(got[:placed], want[0]) and np.array_equal(after, want[1]), i
        assert (got["status"][placed + 1:] == E.ST_GANG_TRIMMED).all()
        trims += 1
    assert trims > 10
    el.close()
    cut.close()


def test_c1_c2_codes_in_every_state():
    """C1: isl_create's codes with the bit; C2: a few-node byte is accepted with the bit, N6's EINVAL stays without it; isl_place_gangs
    keeps its codes in every state (no profiles, no inventory, a snapshot, an empty partition), and isl_preempt keeps P1 (bytes 2 and
    above 3 are EINVAL)."""
    lib = E.load_library()
    M, L = E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED
    for policy, flags, rc in ((M, E.FLAG_GANG_NODE_SCORE_ALL, E.EINVAL), (E.POLICY_FIRST_FIT, ALL | E.FLAG_GANG_FEW_NODES, E.EINVAL),
                              (M, ALL | E.FLAG_ALL_NODES, E.EINVAL), (L, ALL | E.FLAG_GANG_FEW_NODES | E.FLAG_GANG_PREEMPT, E.EINVAL),
                              (L, ALL | E.FLAG_GANG_MIN_MEMBERS | E.FLAG_GANG_PREEMPT, E.EINVAL), (M, ALL | E.FLAG_GANG_BALANCED, E.EINVAL),
                              (M, ALL | E.FLAG_GANG_FEW_NODES | E.FLAG_GANG_ONE_NODE, E.EINVAL),
                              (M, ALL | E.FLAG_GANG_FEW_NODES | E.FLAG_GANG_LOCALITY, E.EINVAL),
                              (M, SCORE | E.FLAG_GANG_FEW_NODES, E.EINVAL), (L, SCORE | E.FLAG_GANG_MIN_MEMBERS, E.EINVAL),
                              (L, SCORE | PER_GANG, E.EINVAL),
                              (M, ALL | E.FLAG_GANG_FEW_NODES, E.OK), (L, ALL | E.FLAG_GANG_MIN_MEMBERS, E.OK),
                              (M, ALL | E.FLAG_GANG_FEW_NODES | E.FLAG_GANG_MIN_MEMBERS, E.OK), (L, ALL | PER_GANG, E.OK),
                              (M, ALL | PER_GANG | E.FLAG_GANG_MIN_MEMBERS | E.FLAG_GANG_PREEMPT, E.EINVAL),
                              (M, ALL | PER_GANG | E.FLAG_GANG_PREEMPT, E.OK), (L, ALL, E.OK)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == rc, (policy, flags)
        if rc == E.OK:
            lib.isl_destroy(h)
    cfg = E.Config(E.ABI_VERSION, M, E.QUIRKS_REF_EXACT, -1, (1 << 20) + 1, 16, ALL | E.FLAG_GANG_FEW_NODES, 0)
    assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(ctypes.c_void_p())) == E.ERANGE
    rows = E.make_profiles(tables.A100_40GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off, r=req):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(r), p(out))

    few = req.copy()
    few["start"] = E.GANG_FEW_NODES
    bad = few.copy()
    bad["start"][1] = 9                                          # a balanced byte on an engine without BALANCED, then two bytes
    fresh = E.Engine(max_gpus=16, max_batch=16, policy=M, flags=ALL | E.FLAG_GANG_LOCALITY)
    assert call(fresh, [0, 1]) == E.ESTATE
    assert call(fresh, [0, 2], bad) == E.EINVAL                  # L4 comes before the state
    fresh.load_profiles(rows)
    assert call(fresh, [0, 2], few) == E.ESTATE                  # a few-node byte passes the argument checks with the bit
    eng = engine(node_offsets(2, 2), rows, np.array([0x01, 0, 0, 0], dtype=np.uint8), M, ALL | E.FLAG_GANG_LOCALITY, max_batch=3)
    assert call(eng, [0, 4]) == E.ERANGE
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL
    eng.snapshot_occupancy()
    eng.reset_stats()
    before = (eng.read_occupancy().tolist(), eng.stats())
    assert call(eng, [0, 2], bad[:2]) == E.EINVAL
    assert (eng.read_occupancy().tolist(), eng.stats()) == before
    assert eng.restore_occupancy() is None                       # the snapshot is still there
    assert call(eng, [0, 3], few[:3]) == E.OK and out["status"][:3].tolist() == [E.ST_PLACED] * 3
    eng.set_partition(1, 1)
    assert call(eng, [0, 1]) == E.ERANGE
    eng.close()
    pre = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), L, ALL | E.FLAG_GANG_LOCALITY | E.FLAG_GANG_PREEMPT)
    prio = np.full(2, 5, dtype=np.uint8)
    for b in (E.GANG_FEW_NODES, 4):
        with pytest.raises(E.EngineError):                       # P1: isl_preempt refuses bytes 2 and above 3 with the bit too
            pre.preempt(req[:2], prio, np.zeros(0, dtype=E.VICTIM_DTYPE), gang_off=[0, 2], locality=[b])
    with pytest.raises(E.EngineError):                           # node scoring opens no stream (rule 7), with the bit as without
        pre.stream_open(1)
    pre.close()
    fresh.close()


def test_worked_examples():
    """The header's C4 example: MOST_ALLOCATED few-node rounds take node 1 then node 2; LEAST_ALLOCATED node 0 then node 1."""
    rows = E.make_profiles(tables.H100_80GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    for policy, want in ((E.POLICY_MOST_ALLOCATED, [(1, 0), (1, 1), (1, 2), (2, 6)]), (E.POLICY_LEAST_ALLOCATED, [(0, 4), (0, 5), (0, 6), (1, 0)])):
        eng = engine(np.arange(4, dtype=np.uint32), rows, np.array([0x0F, 0xF8, 0x3F], dtype=np.uint8), policy, ALL | E.FLAG_GANG_FEW_NODES)
        assert [(int(r["gpu"]), int(r["start"])) for r in eng.place_gangs(req, [0, 4])] == want
        eng.close()


def test_place_pending_gangs_score_all():
    """A reconciler with every gang kind scored: a few-node job whose second round joins the fuller node under MostAllocated and the
    emptier one under LeastAllocated, and elastic distinct-node replicas placed with their leading pods."""
    for policy in POLICIES:
        r = ctl.InstasliceReconciler(cr_cluster([1, 1, 1]), policy=policy, gang_node_score=True, gang_node_score_all=True,
                                     gang_locality=True, gang_min_members=True)
        out = r.place_pending_gangs([pods(["1g.5gb"], "a"), pods(["1g.5gb"] * 9, "b"), pods(["1g.5gb"] * 4, "c")],
                                    locality=[E.GANG_ANY_NODES, E.GANG_FEW_NODES, E.GANG_DISTINCT_NODES], min_members=[0, 0, 1])
        assert [v for v, _ in out] == ["placed", "placed", "placed"]
        assert out[0][1][0]["nodename"] == "node-0"
        assert [a["nodename"] for a in out[1][1][:7]] == ["node-1"] * 7
        assert {a["nodename"] for a in out[1][1][7:]} == {"node-0" if policy == E.POLICY_MOST_ALLOCATED else "node-2"}
        # elastic replicas on distinct nodes: node-1 is full, so the leading two are placed, on node-0 (the fuller under MostAllocated,
        # the emptier under LeastAllocated) and node-2
        assert [a["nodename"] for a in out[2][1]] == ["node-0", "node-2"]
        plain = ctl.InstasliceReconciler(cr_cluster([1, 1]), policy=policy, gang_node_score=True, gang_node_score_all=True,
                                         gang_few_nodes=True)
        assert plain.place_pending_gangs([pods(["1g.5gb"] * 9, "d")])[0][0] == "placed"


def test_host_mirror_gang_score_all_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_score_all_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_score_all_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
