"""Elastic gangs (isl_place_gangs on an engine created with ISL_FLAG_GANG_MIN_MEMBERS) on the H100: k_ganglocal<true> against the direct
brute force tests/gang_min_fast.cpp, records, final occupancy and stats.placed byte-identical, under every policy, both quirk sets and
every gang flag (none, one node, few nodes, distinct nodes, locality per gang); the hand-worked vectors; M5 (a), (b) and (d) device
against device; the M6 refusals and the isl_place_gangs codes in every engine state; the table, inventory and layout limits; a gang of
300 members trimmed past its 256th; the reconciler flow and the C++ host mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_min_fast as GMF
import gang_min_oracle as GMO
import gang_oracle as GO
from test_gpu_gang_few import cluster, cr_cluster, device, pods, random_call
from test_oracle_gang_topology_limits import CASES, FIXTURES, LAYOUT_CASES, case_ids, gang_plan, layout_cases, lower_half_full, small_gangs
from test_oracle_request_major_limits import eight_gpu_nodes, gang_call, node_tables_for, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
MIN = E.FLAG_GANG_MIN_MEMBERS
# every gang flag with MIN: (name, engine flags, locality of every gang; None = a random locality per gang)
MODES = [("any", 0, E.GANG_ANY_NODES), ("one", E.FLAG_GANG_ONE_NODE, E.GANG_ONE_NODE), ("few", E.FLAG_GANG_FEW_NODES, E.GANG_FEW_NODES),
         ("distinct", E.FLAG_GANG_DISTINCT_NODES, E.GANG_DISTINCT_NODES), ("locality", E.FLAG_GANG_LOCALITY, None)]


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=MIN):
    eng = E.Engine(max_gpus=max(4097, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if np.asarray(rows).ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def minima_for(rng, off, most=8):
    return (rng.next(len(off) - 1) % np.uint64(most + 1)).astype(np.int64)


def check(eng, rows, node_off, node_table, occ, req, off, mode_flags, locality, minima, policy, quirks, part=None, what=""):
    """Load the inventory (and the partition) into ``eng``, place the call with ``minima`` (and ``locality`` per gang on a locality
    engine), compare records, occupancy and stats.placed with the brute force."""
    G = int(node_off[-1])
    lo, hi = part or (0, G)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    if part:
        eng.set_partition(lo, hi)
    want, occ_want, placed = GMF.place_gangs(node_off, rows, occ, GMO.with_minimum(req, off, minima), off, locality, quirks, policy,
                                             node_table, lo, hi)
    eng.reset_stats()
    got = eng.place_gangs(req, off, locality if mode_flags & E.FLAG_GANG_LOCALITY else None, minima)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    assert eng.stats()["placed"] == placed, what
    return got


def mode_locality(rng, mode, n_gangs):
    _name, _flags, loc = mode
    return (rng.next(n_gangs) % np.uint64(4)).astype(np.int64) if loc is None else np.full(n_gangs, loc, dtype=np.int64)


@pytest.mark.parametrize("kat", list(GMO.load_kat()), ids=lambda k: k[0])
def test_kat(kat):
    _name, inp, req, off, want, occ_after, placed = kat
    eng = engine(inp["node_off"], inp["rows"], inp["occ"], inp["policy"], inp["quirks"], inp["node_table"], flags=MIN | E.FLAG_GANG_LOCALITY)
    if inp["partition"]:
        eng.set_partition(*inp["partition"])
    eng.reset_stats()
    assert [tuple(int(x) for x in r) for r in eng.place_gangs(req, off)] == want
    assert eng.read_occupancy().tolist() == occ_after.tolist()
    assert eng.stats()["placed"] == placed
    eng.close()


@pytest.mark.parametrize("mode", MODES, ids=[m[0] for m in MODES])
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("policy", POLICIES)
def test_vs_brute_force(policy, quirks, mode):
    """Nodes of 0 to 16 GPUs (empty ones among them), gangs of 1..12 with FREEs, NOOPs and unknown profiles between the members, random
    minima, whole and cut partitions."""
    rng = SplitMix64(12100 + policy * 100 + quirks * 10 + MODES.index(mode))
    outcomes = set()
    for trial in range(3):
        sizes = [int(rng.next1() % 17) for _ in range(120)]
        node_off, rows, occ, node_table, n_names = cluster(rng, 1 + 2 * (trial % 2), sizes, 0x7F if trial % 2 else 0xFF)
        G = int(node_off[-1])
        req, off = random_call(rng, G, n_names, 500 if policy == E.POLICY_MIN_FRAG else 1200, 12)
        part = None if trial < 2 else (int(rng.next1() % (G // 3)), G - int(rng.next1() % (G // 3)))
        eng = engine(node_off, rows, occ, policy, quirks, node_table, flags=MIN | mode[1])
        got = check(eng, rows, node_off, node_table, occ, req, off, mode[1], mode_locality(rng, mode, len(off) - 1), minima_for(rng, off),
                    policy, quirks, part, what=trial)
        eng.close()
        outcomes |= set(np.unique(got["status"]).tolist())
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_GANG_TRIMMED, E.ST_NO_CAPACITY} <= outcomes


@pytest.mark.parametrize("mode", MODES, ids=[m[0] for m in MODES])
@pytest.mark.parametrize("policy", POLICIES)
def test_m5a_equals_unflagged(policy, mode):
    """M5 (a), device against device: with every byte 0, or every byte at least its gang's k, a MIN engine equals the engine without
    MIN: records, occupancy and stats.placed."""
    rng = SplitMix64(12300 + policy * 10 + MODES.index(mode))
    node_off, rows, occ, node_table, n_names = cluster(rng, 3, [int(rng.next1() % 9) for _ in range(200)], 0x7F)
    G = int(node_off[-1])
    req, off = random_call(rng, G, n_names, 1200, 10)
    locality = mode_locality(rng, mode, len(off) - 1)
    per_gang = locality if mode[1] & E.FLAG_GANG_LOCALITY else None
    k = np.add.reduceat(req["op"] == E.OP_ALLOC, off[:-1].astype(np.int64)).astype(np.int64)
    part = (int(rng.next1() % 40), G - int(rng.next1() % 40))
    b = engine(node_off, rows, occ, policy, E.QUIRKS_REF_EXACT, node_table, flags=mode[1])
    b.set_partition(*part)
    b.reset_stats()
    want = b.place_gangs(req, off, per_gang)
    for minima in (np.zeros(len(k), np.int64), np.minimum(255, k + (rng.next(len(k)) % np.uint64(3)).astype(np.int64))):
        a = engine(node_off, rows, occ, policy, E.QUIRKS_REF_EXACT, node_table, flags=MIN | mode[1])
        a.set_partition(*part)
        a.reset_stats()
        assert np.array_equal(a.place_gangs(req, off, per_gang, minima), want)
        assert np.array_equal(a.read_occupancy(), b.read_occupancy())
        assert a.stats()["placed"] == b.stats()["placed"]
        a.close()
    b.close()


@pytest.mark.parametrize("mode", MODES[:4], ids=[m[0] for m in MODES[:4]])
@pytest.mark.parametrize("policy", POLICIES)
def test_m5b_trimmed_equals_cut_gang(policy, mode):
    """M5 (b), device against device: the call gang by gang on a MIN engine, beside an engine without MIN that places each trimmed gang
    cut to its first f ALLOC members (and every other gang whole): the cut gang commits with the same records, and the occupancies
    agree after every gang."""
    rng = SplitMix64(12500 + policy * 10 + MODES.index(mode))
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(60)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = (rng.next(G) & np.uint64(0xBF)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 500, 10)
    req["op"][req["op"] != E.OP_ALLOC] = E.OP_NOOP
    minima = minima_for(rng, off, 6)
    a, b = engine(node_off, rows, occ, policy, flags=MIN | mode[1]), engine(node_off, rows, occ, policy, flags=mode[1])
    trimmed = 0
    for g, (lo, hi) in enumerate(zip(off[:-1], off[1:])):
        idx = np.flatnonzero(req["op"][lo:hi] == E.OP_ALLOC) + lo
        if len(idx) == 0:
            continue
        got = a.place_gangs(req[idx], [0, len(idx)], None, [minima[g]])
        f = int((got["status"] == E.ST_PLACED).sum())
        if 0 < f < len(idx):
            assert (got["status"][:f] == E.ST_PLACED).all() and (got["status"][f + 1:] == E.ST_GANG_TRIMMED).all()
            cut = b.place_gangs(req[idx[:f]], [0, f])
            assert np.array_equal(cut, got[:f]), g
            trimmed += 1
        else:
            b.place_gangs(req[idx], [0, len(idx)])
        assert np.array_equal(a.read_occupancy(), b.read_occupancy()), g
    assert trimmed > 0
    a.close()
    b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_m5d_gangs_of_one(policy):
    """M5 (d): gangs of one ALLOC member with any byte give the records and occupancy of the engine without MIN, for every gang flag."""
    rng = SplitMix64(12700 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 8) for _ in range(200)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 1500, 1)
    minima = (rng.next(len(off) - 1) % np.uint64(256)).astype(np.int64)
    for _name, flags, _loc in MODES[:4]:
        a, b = engine(node_off, rows, occ, policy, flags=MIN | flags), engine(node_off, rows, occ, policy, flags=flags)
        assert np.array_equal(a.place_gangs(req, off, None, minima), b.place_gangs(req, off)), flags
        assert np.array_equal(a.read_occupancy(), b.read_occupancy()), flags
        a.close()
        b.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_gang_of_300_trimmed_past_256(policy):
    """One gang of 300 7g.80gb (a whole GPU each under fixed quirks) with m = 255 on 270 empty GPUs: every locality that can take 270
    stops at f = 270 >= 255 and writes TRIMMED for ranks 271..299, past several blocks of 32; the one-node gang sits on one node of 270
    GPUs.  Distinct-node gangs get 270 one-GPU nodes too."""
    rows = E.make_profiles(tables.H100_80GB)
    p7 = [r[0] for r in tables.H100_80GB].index("7g.80gb")
    req = alloc_requests(np.full(300, p7, dtype=np.uint8))
    off = np.array([0, 300], dtype=np.uint32)
    for loc, node_off in ((E.GANG_ANY_NODES, node_offsets(270, 1)), (E.GANG_FEW_NODES, node_offsets(270, 1)),
                          (E.GANG_DISTINCT_NODES, node_offsets(270, 1)), (E.GANG_ONE_NODE, np.array([0, 5, 275, 280], dtype=np.uint32))):
        G = int(node_off[-1])
        occ = np.zeros(G, dtype=np.uint8)
        if loc == E.GANG_ONE_NODE:
            occ[:5] = occ[275:] = 0xFF                  # only the middle node has room
        eng = engine(node_off, rows, occ, policy, E.QUIRKS_FIXED, flags=MIN | E.FLAG_GANG_LOCALITY, max_batch=300)
        got = check(eng, rows, node_off, None, occ, req, off, E.FLAG_GANG_LOCALITY, [loc], [255], policy, E.QUIRKS_FIXED, what=loc)
        assert (got["status"][:270] == E.ST_PLACED).all() and got["status"][270] == E.ST_NO_CAPACITY, loc
        assert (got["status"][271:] == E.ST_GANG_TRIMMED).all() and eng.stats()["placed"] == 270, loc
        eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_table_limits(name, quirks, policy):
    """16 profiles and 8 node tables on 4 096 / 4 097 GPUs of eight-GPU nodes, whole bytes, random localities and minima."""
    rows = FIXTURES[name]()
    rng = SplitMix64(13300 + 10 * policy + quirks + len(name))
    n = 300 if policy == E.POLICY_MIN_FRAG else 800
    eng = E.Engine(max_gpus=4097, max_batch=1 << 16, policy=policy, quirks=quirks, flags=MIN | E.FLAG_GANG_LOCALITY)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    for G in (4096, 4097):
        node_off = eight_gpu_nodes(G)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        off = small_gangs(rng, n, 8)
        check(eng, rows, node_off, node_table, whole_bytes(rng, G, dense=True), gang_call(rng, G, rows.shape[-1], n), off,
              E.FLAG_GANG_LOCALITY, (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64), minima_for(rng, off, 5), policy, quirks,
              what=G)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy):
    """T8tab on 2^20 GPUs with node tables and the lower half full; under right-to-left also the top partition, which cuts a node."""
    G = 1 << 20
    rng = SplitMix64(G + policy + 17)
    rows, node_off, node_table, occ, req, off = lower_half_full(rng, G, 100 if policy == E.POLICY_MIN_FRAG else 160)
    eng = E.Engine(max_gpus=G, max_batch=1 << 16, policy=policy, quirks=E.QUIRKS_FIXED, flags=MIN | E.FLAG_GANG_LOCALITY)
    eng.load_profile_tables(rows)
    loc = (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64)
    got = check(eng, rows, node_off, node_table, occ, req, off, E.FLAG_GANG_LOCALITY, loc, minima_for(rng, off, 3), policy, E.QUIRKS_FIXED,
                what="2^20")
    assert (got["gpu"][(got["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)] >= G // 2).any()
    if policy == E.POLICY_RIGHT_TO_LEFT:
        lo = G - 4096 - 13
        req = gang_call(rng, G, 16, 400)
        off = small_gangs(rng, 400)
        got = check(eng, rows, node_off, node_table, whole_bytes(rng, G), req, off, E.FLAG_GANG_LOCALITY,
                    (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64), minima_for(rng, off, 3), policy, E.QUIRKS_FIXED,
                    part=(lo, G), what="top")
        assert (got["status"] == E.ST_PLACED).any() and (got["gpu"][got["status"] == E.ST_PLACED] >= lo).all()
    eng.close()


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_edges(case):
    """Every edge of the CTA layout built from this device's SM count and k_ganglocal's shared-memory opt-in, shares on both sides of the
    shared / global memory switch among them, on an engine without a locality flag (every gang through locality 0)."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    assert edge(gang_plan(node_off, lo, hi, sms, optin - 256)), case
    i = LAYOUT_CASES.index(case)
    policy = (E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT)[i % 3]
    rows = t8tab()
    rng = SplitMix64(480 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    eng = E.Engine(max_gpus=max(4097, G), max_batch=1 << 16, policy=policy, quirks=E.QUIRKS_FIXED, flags=MIN)
    eng.load_profile_tables(rows)
    part = None if (lo, hi) == (0, G) else (lo, hi)
    off = small_gangs(rng, 400, 8)
    got = check(eng, rows, node_off, node_table, whole_bytes(rng, G, dense=True), gang_call(rng, G, 16, 400), off, 0, E.GANG_ANY_NODES,
                minima_for(rng, off, 4), policy, E.QUIRKS_FIXED, part, what=case)
    assert (got["status"] == E.ST_PLACED).any()
    eng.close()


def test_global_memory_share():
    """One node of 2^20 GPUs, whose share lives in global memory, under every locality with minima."""
    G = 1 << 20
    rng = SplitMix64(G + 99)
    node_off = node_offsets(1, G)
    rows = E.make_profiles(tables.H100_80GB)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 64, 24)
    eng = engine(node_off, rows, occ, E.POLICY_FIRST_FIT, max_batch=64, flags=MIN | E.FLAG_GANG_LOCALITY)
    check(eng, rows, node_off, None, occ, req, off, E.FLAG_GANG_LOCALITY, (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64),
          minima_for(rng, off, 12), E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT)
    eng.close()


def test_refusals_and_states():
    """M6: the isl_create refusals and acceptances; EINVAL with nothing changed for two bytes in one gang, before the engine state is
    looked at; a FREE's size is its span and a NOOP's is ignored; isl_place_gangs keeps its codes in every state; Engine.place_gangs's
    argument checks."""
    lib = E.load_library()
    for policy, flags in ((E.POLICY_FIRST_FIT, MIN | E.FLAG_ALL_NODES), (E.POLICY_MOST_ALLOCATED, MIN), (E.POLICY_LEAST_ALLOCATED, MIN),
                          (E.POLICY_FIRST_FIT, MIN | E.FLAG_GANG_ONE_NODE | E.FLAG_GANG_DISTINCT_NODES),
                          (E.POLICY_FIRST_FIT, MIN | E.FLAG_GANG_LOCALITY | E.FLAG_GANG_FEW_NODES)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == E.EINVAL, (policy, flags)
    for _name, flags, _loc in MODES:                        # the flag alone or with exactly one of the four
        E.Engine(max_gpus=16, max_batch=16, flags=MIN | flags).close()
    rows = E.make_profiles(tables.A100_40GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off, r=req):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(r), p(out))

    mixed = req.copy()
    mixed["size"] = [1, 2, 1, 1]
    fresh = E.Engine(max_gpus=16, max_batch=16, flags=MIN)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no profiles
    assert call(fresh, [0, 2], mixed) == E.EINVAL                # M6 comes before the state
    fresh.load_profiles(rows)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no inventory
    eng = engine(node_offsets(2, 2), rows, np.array([0x01, 0, 0, 0], dtype=np.uint8), max_batch=3)
    assert call(eng, [0, 4]) == E.ERANGE
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL
    assert call(eng, [1, 3]) == E.EINVAL
    assert lib.isl_place_gangs(eng._h, 1, None, p(req), p(out)) == E.EINVAL
    assert call(eng, [0]) == E.OK
    eng.snapshot_occupancy()
    eng.reset_stats()
    before = (eng.read_occupancy().tolist(), eng.stats())
    for sizes, off in (([1, 2, 1], [0, 3]), ([0, 3, 2], [0, 1, 3]), ([5, 5, 0], [0, 3]), ([0, 255, 254], [0, 1, 3])):
        bad = req[:3].copy()
        bad["size"] = sizes
        assert call(eng, off, bad) == E.EINVAL, sizes
    assert (eng.read_occupancy().tolist(), eng.stats()) == before
    assert eng.restore_occupancy() is None                       # the snapshot is still there
    ok = req[:3].copy()
    ok["handle"][1], ok["op"][1], ok["start"][1], ok["size"][1] = 0, E.OP_FREE, 0, 1     # a FREE's size is its span: slice 0 of GPU 0
    ok["op"][2], ok["size"][2] = E.OP_NOOP, 200
    ok["size"][0] = 7
    assert call(eng, [0, 3], ok) == E.OK and out["status"][:3].tolist() == [E.ST_PLACED, E.ST_FREED, E.ST_NOOP]
    assert out["gpu"][0] == 0 and out["start"][0] == 0            # the FREE came first
    eng.set_partition(1, 1)
    assert call(eng, [0, 1]) == E.ERANGE                         # an empty partition
    eng.close()
    eng = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8))
    eng.stream_open(1)
    try:
        assert call(eng, [0, 1]) == E.ESTATE                     # an open stream owns the engine
    finally:
        eng.stream_close()
    assert call(eng, [0, 2]) == E.OK
    for bad_min in ([1], [-1, 0], [256, 0]):
        with pytest.raises(ValueError):
            eng.place_gangs(req, [0, 2, 4], None, bad_min)
    with pytest.raises(ValueError):
        engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), flags=0).place_gangs(req, [0, 4], None, [1])
    eng.close()
    big = engine(node_offsets(1, (1 << 20) + 8), rows, np.zeros((1 << 20) + 8, dtype=np.uint8))
    assert call(big, [0, 1]) == E.ERANGE                         # a partition of more than 2^20 GPUs
    big.set_partition(8, (1 << 20) + 8)
    assert call(big, [0, 2]) == E.OK and out["gpu"][:2].tolist() == [8, 8]
    big.close()
    fresh.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_other_calls_unchanged(policy):
    """M6: every other call on a MIN engine returns what it returns on an unflagged one, whatever the requests' size bytes."""
    rng = SplitMix64(13005 + policy)
    node_off = node_offsets(500, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(4000) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, 4000, len(rows), 5000, 1)
    alloc = req["op"] == E.OP_ALLOC
    req["size"][alloc] = (rng.next(int(alloc.sum())) % np.uint64(256)).astype(np.uint8)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=0)
    assert np.array_equal(a.place_batch(req), b.place_batch(req))
    assert np.array_equal(a.place_batch_range(800, 1600, req), b.place_batch_range(800, 1600, req))
    assert np.array_equal(a.read_occupancy(), b.read_occupancy())
    a.close()
    b.close()


def test_place_pending_gangs_min_members():
    """Three one-GPU nodes: a gang of four 4g.20gb with minimum 2 is placed with its first three pods (only their allocations are
    written), a gang of ten 1g.5gb where nine fit is not placed, and the engine and the custom resources agree after the call."""
    items = cr_cluster([1, 1, 1])
    r = ctl.InstasliceReconciler(items, gang_min_members=True)
    out = r.place_pending_gangs([pods(["4g.20gb"] * 4, "a"), pods(["1g.5gb"] * 10, "b"), pods(["1g.5gb", "1g.5gb"], "c")],
                                min_members=[2, 0, 0])
    assert [v for v, _ in out] == ["placed", "none", "placed"]
    assert [a["nodename"] for a in out[0][1]] == ["node-0", "node-1", "node-2"]
    assert [(a["nodename"], a["start"]) for a in out[2][1]] == [("node-0", 4), ("node-0", 5)]
    assert not any("a3" in it["spec"]["allocations"] for it in items)
    assert np.array_equal(r.engine.read_occupancy(), GO.cr_occupancy(items))
    with pytest.raises(ValueError):                              # a minimum needs a reconciler created with gang_min_members
        ctl.InstasliceReconciler(cr_cluster([1])).place_pending_gangs([pods(["1g.5gb"], "d")], min_members=[1])


def test_host_mirror_gang_min_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_min_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_min_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
