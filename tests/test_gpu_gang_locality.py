"""Node locality per gang (isl_place_gangs on an engine created with ISL_FLAG_GANG_LOCALITY) on the H100: k_ganglocal against composition
(i) of tests/gang_locality_oracle.py (each run of gangs on the brute force of its locality), records, final occupancy and stats.placed
byte-identical, plus the hand-worked vectors, L3 (a) and (b) device against device, the marks and dead-profile hazards, the L4 / L5
refusals, the isl_place_gangs codes in every engine state, the reconciler flow and the C++ host mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_locality_oracle as GLO
import gang_oracle as GO
from test_gpu_gang_few import cluster, cr_cluster, device, pods, random_call
from test_oracle_gang_topology_limits import CASES, FIXTURES, LAYOUT_CASES, case_ids, gang_plan, layout_cases, lower_half_full, small_gangs
from test_oracle_request_major_limits import eight_gpu_nodes, gang_call, node_tables_for, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
LOC = E.FLAG_GANG_LOCALITY


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=LOC):
    eng = E.Engine(max_gpus=max(4097, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if np.asarray(rows).ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def random_localities(rng, n_gangs):
    return (rng.next(n_gangs) % np.uint64(4)).astype(np.int64)


def check(eng, rows, node_off, node_table, occ, req, off, locality, policy, quirks, part=None, what=""):
    """Load the inventory (and the partition) into ``eng``, place the call with ``locality``, compare records, occupancy and
    stats.placed with composition (i)."""
    G = int(node_off[-1])
    lo, hi = part or (0, G)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    if part:
        eng.set_partition(lo, hi)
    want, occ_want = GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(req, off, locality), off, quirks, policy, node_table,
                                             lo, hi)
    eng.reset_stats()
    got = eng.place_gangs(req, off, locality)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    placed = int(((want["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)).sum())
    assert eng.stats()["placed"] == placed, what
    return got


@pytest.mark.parametrize("kat", list(GLO.load_kat()), ids=lambda k: k[0])
def test_kat(kat):
    _name, inp, req, off, want, occ_after = kat
    eng = engine(inp["node_off"], inp["rows"], inp["occ"], inp["policy"], inp["quirks"], inp["node_table"])
    if inp["partition"]:
        eng.set_partition(*inp["partition"])
    assert [tuple(int(x) for x in r) for r in eng.place_gangs(req, off)] == want
    assert eng.read_occupancy().tolist() == occ_after.tolist()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_vs_composition(policy, quirks, n_tables):
    """Nodes of 0 to 16 GPUs (empty ones among them), random localities, gangs of 1..12 with FREEs, NOOPs and unknown profiles between
    the members, whole and cut partitions."""
    rng = SplitMix64(8100 + policy * 100 + quirks * 10 + n_tables)
    outcomes = set()
    for trial in range(4):
        sizes = [int(rng.next1() % 17) for _ in range(150)]
        node_off, rows, occ, node_table, n_names = cluster(rng, n_tables, sizes, 0x7F if trial % 2 else 0xFF)
        G = int(node_off[-1])
        req, off = random_call(rng, G, n_names, 600 if policy == E.POLICY_MIN_FRAG else 1500, 12)
        part = None if trial < 2 else (int(rng.next1() % (G // 3)), G - int(rng.next1() % (G // 3)))
        eng = engine(node_off, rows, occ, policy, quirks, node_table)
        got = check(eng, rows, node_off, node_table, occ, req, off, random_localities(rng, len(off) - 1), policy, quirks, part)
        eng.close()
        outcomes |= set(np.unique(got["status"]).tolist())
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_FREED, E.ST_NOOP, E.ST_BAD_PROFILE} <= outcomes


@pytest.mark.parametrize("policy", POLICIES)
def test_every_pair_of_localities(policy):
    """All 16 ordered pairs of consecutive localities, each pair many times, on one-, two- and four-GPU nodes."""
    rng = SplitMix64(8300 + policy)
    rows = E.make_profiles(tables.A100_40GB)
    node_off = np.cumsum([0] + [(1, 2, 4)[i % 3] for i in range(90)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    pairs = [(a, b) for a in range(4) for b in range(4)]
    locality = np.asarray([x for _ in range(6) for p in pairs for x in p], dtype=np.int64)
    n_gangs = len(locality)
    sizes = 1 + (rng.next(n_gangs) % np.uint64(4)).astype(np.int64)
    off = np.cumsum([0] + sizes.tolist()).astype(np.uint32)
    req = alloc_requests((rng.next(int(off[-1])) % np.uint64(len(rows))).astype(np.uint8))
    eng = engine(node_off, rows, occ, policy)
    got = check(eng, rows, node_off, None, occ, req, off, locality, policy, E.QUIRKS_REF_EXACT)
    assert (got["status"] == E.ST_PLACED).any() and (got["status"] == E.ST_GANG_ABORTED).any()
    eng.close()


@pytest.mark.parametrize("shape", [(1, 1), (3, 4096), (4096, 1), (1024, 8), (131072, 8), (1, 1 << 20)], ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_scale(shape, policy):
    """Inventories from one GPU to 2^20 GPUs, one node of 2^20 GPUs whose share lives in global memory, and a gang of max_batch members
    under each locality."""
    n_nodes, per = shape
    G = n_nodes * per
    rng = SplitMix64(G + policy + 29)
    node_off = node_offsets(n_nodes, per)
    rows = E.make_profiles(tables.H100_80GB)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    n = 64 if G > 65536 else 256
    req, off = random_call(rng, G, len(rows), n, 24)
    eng = engine(node_off, rows, occ, policy, max_batch=n)
    check(eng, rows, node_off, None, occ, req, off, random_localities(rng, len(off) - 1), policy, E.QUIRKS_REF_EXACT)
    for loc in GLO.LOCALITIES:
        check(eng, rows, node_off, None, occ, req, np.array([0, n], dtype=np.uint32), [loc], policy, E.QUIRKS_REF_EXACT, what=loc)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_table_limits(name, quirks, policy):
    """16 profiles and 8 node tables on 4 096 / 4 097 GPUs of eight-GPU nodes, whole bytes, random localities."""
    rows = FIXTURES[name]()
    rng = SplitMix64(9300 + 10 * policy + quirks + len(name))
    n = 300 if policy == E.POLICY_MIN_FRAG else 800
    eng = E.Engine(max_gpus=4097, max_batch=1 << 16, policy=policy, quirks=quirks, flags=LOC)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    for G in (4096, 4097):
        node_off = eight_gpu_nodes(G)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        off = small_gangs(rng, n, 8)
        check(eng, rows, node_off, node_table, whole_bytes(rng, G, dense=True), gang_call(rng, G, rows.shape[-1], n), off,
              random_localities(rng, len(off) - 1), policy, quirks, what=G)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy):
    """T8tab on 2^20 GPUs with node tables and the lower half full; under right-to-left also the top partition, which cuts a node."""
    G = 1 << 20
    rng = SplitMix64(G + policy + 11)
    rows, node_off, node_table, occ, req, off = lower_half_full(rng, G, 100 if policy == E.POLICY_MIN_FRAG else 160)
    eng = E.Engine(max_gpus=G, max_batch=1 << 16, policy=policy, quirks=E.QUIRKS_FIXED, flags=LOC)
    eng.load_profile_tables(rows)
    got = check(eng, rows, node_off, node_table, occ, req, off, random_localities(rng, len(off) - 1), policy, E.QUIRKS_FIXED, what="2^20")
    assert (got["gpu"][(got["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)] >= G // 2).any()
    if policy == E.POLICY_RIGHT_TO_LEFT:
        lo = G - 4096 - 13
        req = gang_call(rng, G, 16, 400)
        off = small_gangs(rng, 400)
        got = check(eng, rows, node_off, node_table, whole_bytes(rng, G), req, off, random_localities(rng, len(off) - 1), policy,
                    E.QUIRKS_FIXED, part=(lo, G), what="top")
        assert (got["status"] == E.ST_PLACED).any() and (got["gpu"][got["status"] == E.ST_PLACED] >= lo).all()
    eng.close()


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_edges(case):
    """Every edge of the CTA layout built from this device's SM count and k_ganglocal's own shared-memory opt-in (its 256 B of static
    shared memory), shares on both sides of the shared / global memory switch among them."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    assert edge(gang_plan(node_off, lo, hi, sms, optin - 256)), case
    i = LAYOUT_CASES.index(case)
    policy = (E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT)[i % 3]
    rows = t8tab()
    rng = SplitMix64(380 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    eng = E.Engine(max_gpus=max(4097, G), max_batch=1 << 16, policy=policy, quirks=E.QUIRKS_FIXED, flags=LOC)
    eng.load_profile_tables(rows)
    part = None if (lo, hi) == (0, G) else (lo, hi)
    off = small_gangs(rng, 400, 8)
    got = check(eng, rows, node_off, node_table, whole_bytes(rng, G, dense=True), gang_call(rng, G, 16, 400), off,
                random_localities(rng, len(off) - 1), policy, E.QUIRKS_FIXED, part, what=case)
    assert (got["status"] == E.ST_PLACED).any()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_each_locality_equals_its_engine(policy, quirks):
    """L3 (a), device against device: a call whose gangs all carry locality k equals the call on an engine created with k's flag (no
    gang flag for 0): records, occupancy and stats.placed, with node tables and a partition that cuts nodes."""
    rng = SplitMix64(8500 + policy * 3 + quirks)
    node_off, rows, occ, node_table, n_names = cluster(rng, 3, [int(rng.next1() % 9) for _ in range(200)], 0x7F)
    G = int(node_off[-1])
    req, off = random_call(rng, G, n_names, 1500, 10)
    part = (int(rng.next1() % 50), G - int(rng.next1() % 50))
    for loc in GLO.LOCALITIES:
        a, b = engine(node_off, rows, occ, policy, quirks, node_table), engine(node_off, rows, occ, policy, quirks, node_table,
                                                                                flags=GLO.FLAG_OF[loc])
        a.set_partition(*part)
        b.set_partition(*part)
        a.reset_stats()
        b.reset_stats()
        assert np.array_equal(a.place_gangs(req, off, [loc] * (len(off) - 1)), b.place_gangs(req, off)), loc
        assert np.array_equal(a.read_occupancy(), b.read_occupancy()), loc
        assert a.stats()["placed"] == b.stats()["placed"], loc
        a.close()
        b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_gang_by_gang_on_four_engines(policy):
    """L3 (b): a call equals its gangs run one at a time after the call's FREEs, each alone on the engine flagged for its locality, with
    the whole occupancy handed over (isl_read_occupancy, isl_write_occupancy) from each gang to the next."""
    rng = SplitMix64(8700 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(80)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = (rng.next(G) & np.uint64(0xBF)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 600, 8)
    locality = random_localities(rng, len(off) - 1)
    one = engine(node_off, rows, occ, policy)
    got = one.place_gangs(req, off, locality)
    engines = {loc: engine(node_off, rows, occ, policy, flags=GLO.FLAG_OF[loc]) for loc in GLO.LOCALITIES}
    frees = req.copy()
    frees["op"][frees["op"] == E.OP_ALLOC] = E.OP_NOOP
    want = engines[0].place_gangs(frees, [0, len(req)])
    cur = engines[0].read_occupancy()
    for g, (a, b) in enumerate(zip(off[:-1], off[1:])):
        alloc = np.flatnonzero(req["op"][a:b] == E.OP_ALLOC) + a
        if len(alloc) == 0:
            continue
        eng = engines[int(locality[g])]
        eng.write_occupancy(0, cur)
        want[alloc] = eng.place_gangs(req[alloc], [0, len(alloc)])
        cur = eng.read_occupancy()
    assert np.array_equal(got, want)
    assert np.array_equal(one.read_occupancy(), cur)
    for eng in [one, *engines.values()]:
        eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_any_node_gangs_of_one_equal_place_batch(policy):
    """L3 (c): with every byte 0, gangs of one equal isl_place_batch."""
    rng = SplitMix64(8800 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 12) for _ in range(300)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, G, len(rows), 3000, 1)
    a, c = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=0)
    assert np.array_equal(a.place_gangs(req, np.arange(len(req) + 1)), c.place_batch(req))
    assert np.array_equal(a.read_occupancy(), c.read_occupancy())
    a.close()
    c.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_marks_after_scratch_copies(policy):
    """More than 255 distinct-node gangs interleaved with one-node and few-node gangs, whose scratch copies overwrite the node-used marks:
    every occupancy byte equals some tag, and a distinct-node gang follows every scratch copy directly."""
    rng = SplitMix64(8900 + policy)
    rows = E.make_profiles(tables.A100_40GB)
    node_off = node_offsets(160, 4)
    G = 640
    occ = ((rng.next(G) % np.uint64(255)) + np.uint64(1)).astype(np.uint8)     # bytes 1..255: the values the tags take
    occ[::2] = 0
    # 300 distinct-node gangs in a row (the tags wrap), then one-node or few-node gangs each followed by two distinct-node gangs
    locality = np.concatenate([np.full(300, E.GANG_DISTINCT_NODES),
                               np.where(np.arange(300) % 3 == 0, (rng.next(300) % np.uint64(2)).astype(np.int64) + 1, E.GANG_DISTINCT_NODES)])
    n_gangs = len(locality)
    sizes = 1 + (rng.next(n_gangs) % np.uint64(2)).astype(np.int64)
    off = np.cumsum([0] + sizes.tolist()).astype(np.uint32)
    req = alloc_requests(np.where(rng.next(int(off[-1])) % np.uint64(4) == 0, 1, 0).astype(np.uint8))     # 1g.5gb, some 2g.10gb
    eng = engine(node_off, rows, occ, policy)
    got = check(eng, rows, node_off, None, occ, req, off, locality, policy, E.QUIRKS_REF_EXACT)
    spread = np.asarray([locality[g] == E.GANG_DISTINCT_NODES and (got["status"][off[g]:off[g + 1]] == E.ST_PLACED).any()
                         for g in range(n_gangs)])
    assert spread.sum() > 255
    eng.close()


def test_dead_bit_only_on_committed_state():
    """A locality-0 gang [p, q] whose q fails only because of p's tentative slice must not mark q dead: the next gang places q.  Fixed
    quirks, where 7g.40gb fits an empty GPU (under the strict bound it fits nowhere)."""
    rows = E.make_profiles(tables.A100_40GB)
    A = {name: i for i, (name, *_rest) in enumerate(tables.A100_40GB)}
    eng = engine(node_offsets(1, 1), rows, np.array([0x00], dtype=np.uint8), quirks=E.QUIRKS_FIXED)
    req = alloc_requests(np.array([A["4g.20gb"], A["7g.40gb"], A["7g.40gb"]], dtype=np.uint8))
    got = eng.place_gangs(req, [0, 2, 3], [E.GANG_ANY_NODES, E.GANG_ANY_NODES])
    assert [tuple(int(x) for x in r) for r in got] == [(E.GPU_NONE, 9, 4, E.ST_GANG_ABORTED), (E.GPU_NONE, 9, 8, E.ST_NO_CAPACITY),
                                                      (0, 0, 8, E.ST_PLACED)]
    for loc in GLO.LOCALITIES:        # the same after a gang of each locality whose first member fails on the committed state
        eng.load_inventory(node_offsets(1, 1), np.array([0x00], dtype=np.uint8))
        req = alloc_requests(np.array([A["4g.20gb"], A["7g.40gb"], A["4g.20gb"], A["7g.40gb"]], dtype=np.uint8))
        got = eng.place_gangs(req, [0, 2, 3, 4], [E.GANG_ANY_NODES, E.GANG_ANY_NODES, loc])
        assert got["status"].tolist() == [E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_PLACED, E.ST_NO_CAPACITY], loc
    eng.close()


def test_refusals_and_states():
    """L4: EINVAL with nothing changed for a byte above 3 or two localities in one gang; L5: the isl_create refusals; isl_place_gangs keeps
    its codes in every state."""
    lib = E.load_library()
    for policy, flags in ((E.POLICY_FIRST_FIT, LOC | E.FLAG_GANG_ONE_NODE), (E.POLICY_FIRST_FIT, LOC | E.FLAG_GANG_DISTINCT_NODES),
                          (E.POLICY_FIRST_FIT, LOC | E.FLAG_GANG_FEW_NODES), (E.POLICY_FIRST_FIT, LOC | E.FLAG_ALL_NODES),
                          (E.POLICY_MOST_ALLOCATED, LOC), (E.POLICY_LEAST_ALLOCATED, LOC)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == E.EINVAL, (policy, flags)
    rows = E.make_profiles(tables.A100_40GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off, r=req):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(r), p(out))

    fresh = E.Engine(max_gpus=16, max_batch=16, flags=LOC)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no profiles
    fresh.load_profiles(rows)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no inventory
    bad = req.copy()
    bad["start"][1] = 4
    assert call(fresh, [0, 2], bad) == E.EINVAL                  # L4 comes before the state
    eng = engine(node_offsets(2, 2), rows, np.array([0x01, 0, 0, 0], dtype=np.uint8), max_batch=3)
    assert call(eng, [0, 4]) == E.ERANGE
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL
    assert call(eng, [1, 3]) == E.EINVAL
    assert lib.isl_place_gangs(eng._h, 1, None, p(req), p(out)) == E.EINVAL
    assert call(eng, [0]) == E.OK
    eng.snapshot_occupancy()
    eng.reset_stats()
    before = (eng.read_occupancy().tolist(), eng.stats())
    for starts, off in (([4, 4, 0], [0, 2, 3]), ([1, 2, 0], [0, 2, 3]), ([0, 0, 255], [0, 1, 3]), ([9, 0, 0], [0, 1, 2, 3])):
        bad = req[:3].copy()
        bad["start"] = starts
        assert call(eng, off, bad) == E.EINVAL, starts
    assert (eng.read_occupancy().tolist(), eng.stats()) == before
    assert eng.restore_occupancy() is None                       # the snapshot is still there
    ok = req[:3].copy()
    ok["op"][1], ok["start"][1], ok["size"][1] = E.OP_FREE, 4, 1  # a FREE's start is its span, a NOOP's is ignored
    ok["op"][2], ok["start"][2] = E.OP_NOOP, 200
    ok["start"][0] = E.GANG_DISTINCT_NODES
    assert call(eng, [0, 3], ok) == E.OK and out["status"][:3].tolist() == [E.ST_PLACED, E.ST_FREED, E.ST_NOOP]
    eng.set_partition(1, 1)
    assert call(eng, [0, 1]) == E.ERANGE                         # an empty partition
    eng = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8))
    eng.stream_open(1)
    try:
        assert call(eng, [0, 1]) == E.ESTATE                     # an open stream owns the engine
    finally:
        eng.stream_close()
    assert call(eng, [0, 2]) == E.OK
    with pytest.raises(ValueError):
        engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), flags=0).place_gangs(req, [0, 4], [1])
    big = engine(node_offsets(1, (1 << 20) + 8), rows, np.zeros((1 << 20) + 8, dtype=np.uint8))
    assert call(big, [0, 1]) == E.ERANGE                         # a partition of more than 2^20 GPUs
    big.set_partition(8, (1 << 20) + 8)
    assert call(big, [0, 2]) == E.OK and out["gpu"][:2].tolist() == [8, 8]
    big.close()
    fresh.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_place_batch_unchanged(policy):
    """L5: every other call on a flagged engine returns what it returns on an unflagged one."""
    rng = SplitMix64(9005 + policy)
    node_off = node_offsets(500, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(4000) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, 4000, len(rows), 5000, 1)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=0)
    assert np.array_equal(a.place_batch(req), b.place_batch(req))
    assert np.array_equal(a.place_batch_range(800, 1600, req), b.place_batch_range(800, 1600, req))
    assert np.array_equal(a.read_occupancy(), b.read_occupancy())
    a.close()
    b.close()


def test_place_pending_gangs_locality():
    """Nodes of one, one and two GPUs: a one-node gang goes to node 2, a distinct-node gang to nodes 0 and 1, an any-node gang after
    them, and a gang with no room commits nothing, in one call."""
    items = cr_cluster([1, 1, 2])
    r = ctl.InstasliceReconciler(items, gang_locality=True)
    out = r.place_pending_gangs([pods(["3g.20gb", "3g.20gb"], "a"), pods(["1g.5gb", "1g.5gb"], "b"), pods(["1g.5gb", "1g.5gb"], "c"),
                                 pods(["7g.40gb"], "d")],
                                locality=[E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, E.GANG_ANY_NODES, E.GANG_ANY_NODES])
    assert [v for v, _ in out] == ["placed", "placed", "placed", "none"]
    assert [a["nodename"] for a in out[0][1]] == ["node-2", "node-2"]
    assert [a["nodename"] for a in out[1][1]] == ["node-0", "node-1"]
    assert [(a["nodename"], a["start"]) for a in out[2][1]] == [("node-0", 1), ("node-0", 2)]
    assert np.array_equal(r.engine.read_occupancy(), GO.cr_occupancy(items))


def test_host_mirror_gang_locality_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_locality_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_locality_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
