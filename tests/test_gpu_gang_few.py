"""Few-node gangs (isl_place_gangs on an engine created with ISL_FLAG_GANG_FEW_NODES) on the H100: k_gangnode<true> against the brute
force of tests/gang_few_fast.cpp, records and final occupancy byte-identical, plus the hand-worked vectors, the identities and refusals
of include/islplace.h (F1-F6), the limits of the profile-table ABI and of the CTA layout, the reconciler flow and the C++ host mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_few_fast as GFF
import gang_few_oracle as GFO
import gang_oracle as GO
from test_oracle_gang_topology_limits import CASES, FIXTURES, LAYOUT_CASES, case_ids, gang_plan, layout_cases, lower_half_full, small_gangs
from test_oracle_request_major_limits import GANG_SHAPES, eight_gpu_nodes, gang_call, gang_offsets, node_tables_for, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
FEW = E.FLAG_GANG_FEW_NODES


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=FEW):
    eng = E.Engine(max_gpus=max(4097, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if np.asarray(rows).ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def records(out):
    return [tuple(int(x) for x in r) for r in out]


def assert_runs_are_rounds(eng, got, req, off, rounds):
    """F4 (e): the maximal same-node runs of every committed gang's ALLOC members (isl_gpu_to_node) are its rounds."""
    for a, b in zip(off[:-1], off[1:]):
        idx = [i for i in range(a, b) if req["op"][i] == E.OP_ALLOC]
        if not idx or got["status"][idx[0]] != E.ST_PLACED:
            continue
        nodes = [eng.gpu_to_node(int(got["gpu"][i])) for i in idx]
        starts = [k for k in range(len(idx)) if k == 0 or nodes[k] != nodes[k - 1]]
        assert starts == [k for k in range(len(idx)) if k == 0 or rounds[idx[k]] != rounds[idx[k - 1]]], (a, b, nodes)


def check(eng, rows, node_off, node_table, occ, req, off, policy, quirks, part=None, what=""):
    """Load the inventory (and the partition) into ``eng``, place the call, compare with the brute force and check F4 (e)."""
    G = int(node_off[-1])
    lo, hi = part or (0, G)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    if part:
        eng.set_partition(lo, hi)
    want, occ_want, rounds = GFF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, rounds=True)
    got = eng.place_gangs(req, off)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    assert_runs_are_rounds(eng, got, req, off, rounds)
    return got, rounds


def random_call(rng, G, n_names, n, max_gang):
    req = alloc_requests((rng.next(n) % np.uint64(n_names)).astype(np.uint8))
    req["profile"][rng.next(n) % np.uint64(41) == 0] = E.PROFILE_UNKNOWN
    for i in np.flatnonzero(rng.next(n) % np.uint64(13) == 0):
        start = int(rng.next1() % 8)
        req[i] = (int(rng.next1() % (G + 2)), 0, E.OP_FREE, start, 1 + int(rng.next1() % (8 - start)))
    req["op"][rng.next(n) % np.uint64(29) == 0] = E.OP_NOOP
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % max_gang)))
    return req, np.asarray(off, dtype=np.uint32)


def cluster(rng, n_tables, node_sizes, density):
    node_off = np.cumsum([0] + list(node_sizes)).astype(np.uint32)
    G, n_nodes = int(node_off[-1]), len(node_sizes)
    occ = (rng.next(G) & np.uint64(density)).astype(np.uint8)
    if n_tables == 1:
        rows, node_table = E.make_profiles(tables.H100_80GB), None
        n_names = len(rows)
    else:
        names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
        node_table = (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8)
        n_names = len(names)
    return node_off, rows, occ, node_table, n_names


@pytest.mark.parametrize("kat", list(GFO.load_kat()), ids=lambda k: k[0])
def test_kat(kat):
    _name, inp, gangs, want, occ_after = kat
    for whole in (False, True):
        eng = engine(inp["node_off"], inp["rows"], inp["occ"], inp["policy"], inp["quirks"], inp["node_table"])
        if inp["partition"]:
            eng.set_partition(*inp["partition"])
        if whole:       # all gangs in one call
            req = alloc_requests(np.asarray([p for g in gangs for p in g], dtype=np.uint8))
            off = np.cumsum([0] + [len(g) for g in gangs]).astype(np.uint32)
            assert records(eng.place_gangs(req, off)) == [r for g in want for r in g]
        else:
            for g, w in zip(gangs, want):
                assert records(eng.place_gangs(alloc_requests(np.asarray(g, dtype=np.uint8)), [0, len(g)])) == w
        assert eng.read_occupancy().tolist() == occ_after.tolist()
        eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_vs_brute_force(policy, quirks, n_tables):
    """Nodes of 0 to 16 GPUs, gangs of 1..12 with FREEs, NOOPs and unknown profiles between the members, whole and cut partitions."""
    rng = SplitMix64(3000 + policy * 100 + quirks * 10 + n_tables)
    outcomes, split = set(), 0
    for trial in range(4):
        sizes = [int(rng.next1() % 17) for _ in range(150)]
        node_off, rows, occ, node_table, n_names = cluster(rng, n_tables, sizes, 0x7F if trial % 2 else 0xFF)
        G = int(node_off[-1])
        req, off = random_call(rng, G, n_names, 600 if policy == E.POLICY_MIN_FRAG else 1500, 12)
        part = None if trial < 2 else (int(rng.next1() % (G // 3)), G - int(rng.next1() % (G // 3)))
        eng = engine(node_off, rows, occ, policy, quirks, node_table)
        got, rounds = check(eng, rows, node_off, node_table, occ, req, off, policy, quirks, part)
        eng.close()
        outcomes |= set(np.unique(got["status"]).tolist())
        split += int((rounds > 0).sum())
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_FREED, E.ST_NOOP} <= outcomes and split > 0


@pytest.mark.parametrize("shape", [(1, 1), (3, 4096), (4096, 1), (1024, 8), (131072, 8), (1 << 20, 1), (1, 1 << 20)],
                         ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_scale(shape, policy):
    """Inventories from one GPU to 2^20 GPUs, and one node of 2^20 GPUs whose share lives in global memory; gangs up to max_batch
    members."""
    n_nodes, per = shape
    G = n_nodes * per
    rng = SplitMix64(G + policy + 17)
    node_off = node_offsets(n_nodes, per)
    rows = E.make_profiles(tables.H100_80GB)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    n = 64 if G > 65536 else 256
    req, off = random_call(rng, G, len(rows), n, 24)
    eng = engine(node_off, rows, occ, policy, max_batch=n)
    check(eng, rows, node_off, None, occ, req, off, policy, E.QUIRKS_REF_EXACT)
    check(eng, rows, node_off, None, occ, req, np.array([0, n], dtype=np.uint32), policy, E.QUIRKS_REF_EXACT)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_one_round_per_member(policy):
    """One free 1g slot per one-GPU node: a gang of k members takes k rounds on k nodes; gangs of 33 and 70 members cross the warp
    width of the member scan, and a gang one member larger than the free slots aborts after every other member was placed."""
    rows = E.make_profiles(tables.A100_40GB)
    G = 200
    node_off = node_offsets(G, 1)
    occ = np.full(G, 0x7E, dtype=np.uint8)          # only slice 0 free
    sizes = [33, 70, 2, 96]                         # 201 members: the last gang aborts at its last member
    req = alloc_requests(np.zeros(sum(sizes), dtype=np.uint8))
    off = np.cumsum([0] + sizes).astype(np.uint32)
    eng = engine(node_off, rows, occ, policy)
    got, rounds = check(eng, rows, node_off, None, occ, req, off, policy, E.QUIRKS_REF_EXACT)
    assert rounds[:33].tolist() == list(range(33)) and rounds[33:103].tolist() == list(range(70))
    assert got["status"][-1] == E.ST_NO_CAPACITY and (got["status"][105:-1] == E.ST_GANG_ABORTED).all()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_frees_and_noops_between_split_members(policy):
    """FREEs and NOOPs between the members of gangs that split over nodes; a FREE inside a gang is applied first and never aborts it."""
    rng = SplitMix64(404 + policy)
    rows = E.make_profiles(tables.A100_40GB)
    node_off = node_offsets(64, 2)
    G = 128
    occ = ((rng.next(G) & rng.next(G)) | np.uint64(0x70)).astype(np.uint8)
    req = alloc_requests((rng.next(600) % np.uint64(3)).astype(np.uint8))
    for i in range(1, 600, 4):
        req[i] = (int(rng.next1() % G), 0, E.OP_FREE, int(rng.next1() % 4), 1) if i % 8 == 1 else (0, 0, E.OP_NOOP, 0, 0)
    off = np.asarray(list(range(0, 600, 20)) + [600], dtype=np.uint32)
    eng = engine(node_off, rows, occ, policy)
    got, rounds = check(eng, rows, node_off, None, occ, req, off, policy, E.QUIRKS_REF_EXACT)
    assert (rounds > 0).any() and (got["status"] == E.ST_GANG_ABORTED).any()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_table_limits(name, quirks, policy):
    """16 profiles and 8 node tables (the fixtures of the table-limit tests) on 4 096 / 4 097 GPUs of eight-GPU nodes, whole bytes."""
    rows = FIXTURES[name]()
    rng = SplitMix64(9100 + 10 * policy + quirks + len(name))
    n = 300 if policy == E.POLICY_MIN_FRAG else 1000
    eng = E.Engine(max_gpus=4097, max_batch=1 << 16, policy=policy, quirks=quirks, flags=FEW)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    for G in (4096, 4097):
        node_off = eight_gpu_nodes(G)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        for shape in GANG_SHAPES:
            occ = whole_bytes(rng, G, dense=True)
            check(eng, rows, node_off, node_table, occ, gang_call(rng, G, rows.shape[-1], n), gang_offsets(rng, shape, n), policy, quirks,
                  what=(G, shape))
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy):
    """T8tab on 2^20 GPUs with node tables and the lower half full; under right-to-left also the top partition, which cuts a node."""
    G = 1 << 20
    rng = SplitMix64(G + policy + 7)
    rows, node_off, node_table, occ, req, off = lower_half_full(rng, G, 120 if policy == E.POLICY_MIN_FRAG else 200)
    eng = E.Engine(max_gpus=G, max_batch=1 << 16, policy=policy, quirks=E.QUIRKS_FIXED, flags=FEW)
    eng.load_profile_tables(rows)
    got, _ = check(eng, rows, node_off, node_table, occ, req, off, policy, E.QUIRKS_FIXED, what="2^20")
    assert (got["gpu"][(got["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)] >= G // 2).any()
    if policy == E.POLICY_RIGHT_TO_LEFT:
        lo = G - 4096 - 13
        occ = whole_bytes(rng, G)
        req = gang_call(rng, G, 16, 400)
        got, _ = check(eng, rows, node_off, node_table, occ, req, small_gangs(rng, 400), policy, E.QUIRKS_FIXED, part=(lo, G), what="top")
        assert (got["status"] == E.ST_PLACED).any() and (got["gpu"][got["status"] == E.ST_PLACED] >= lo).all()
    eng.close()


def device():
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_edges(case):
    """Every edge of the CTA layout built from this device's SM count and shared-memory opt-in, shares on both sides of the shared /
    global memory switch among them."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    for static in (0, 1024):
        assert edge(gang_plan(node_off, lo, hi, sms, optin - static)), (case, static)
    i = LAYOUT_CASES.index(case)
    policy = (E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT)[i % 3]
    rows = t8tab()
    rng = SplitMix64(180 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    occ = whole_bytes(rng, G, dense=True)
    eng = E.Engine(max_gpus=max(4097, G), max_batch=1 << 16, policy=policy, quirks=E.QUIRKS_FIXED, flags=FEW)
    eng.load_profile_tables(rows)
    part = None if (lo, hi) == (0, G) else (lo, hi)
    got, _ = check(eng, rows, node_off, node_table, occ, gang_call(rng, G, 16, 400), small_gangs(rng, 400, 8), policy,
                   E.QUIRKS_FIXED, part, what=case)
    assert (got["status"] == E.ST_PLACED).any()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_one_node_engine_gang_by_gang(policy):
    """F4 (a) and (b) on the device, gang by gang from the same state (isl_write_occupancy resynchronises the engines): a gang a
    GANG_ONE_NODE engine commits gets the same records and occupancy, and a gang that aborts here aborts there."""
    rng = SplitMix64(5150 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(60)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = (rng.next(G) & np.uint64(0xBF)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 500, 10)
    few, one = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=E.FLAG_GANG_ONE_NODE)
    seen = set()
    for a, b in zip(off[:-1], off[1:]):
        alloc = req["op"][a:b] == E.OP_ALLOC
        got_one, got_few = one.place_gangs(req[a:b], [0, b - a]), few.place_gangs(req[a:b], [0, b - a])
        occ_one, occ_few = one.read_occupancy(), few.read_occupancy()
        if alloc.any() and (got_one["status"][alloc] == E.ST_PLACED).all():
            assert np.array_equal(got_few, got_one) and np.array_equal(occ_few, occ_one), a
            seen.add("one")
        elif alloc.any() and not (got_few["status"][alloc] == E.ST_PLACED).all():
            assert np.array_equal(occ_few, occ_one), a
            seen.add("abort")
        elif alloc.any():
            seen.add("split")
        one.write_occupancy(0, occ_few)
    assert seen == {"one", "abort", "split"}
    few.close()
    one.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_one_node_equals_unflagged(policy, quirks):
    """F4 (c): a one-node inventory, and a partition inside one node of a larger inventory, give the unflagged engine's answer."""
    rng = SplitMix64(4000 + policy * 3 + quirks)
    rows = E.make_profiles(tables.H100_80GB)
    for node_off, part in ((node_offsets(1, 700), None), (node_offsets(8, 100), (310, 377))):
        G = int(node_off[-1])
        occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
        req, off = random_call(rng, G, len(rows), 1200, 30)
        a, b = engine(node_off, rows, occ, policy, quirks), engine(node_off, rows, occ, policy, quirks, flags=0)
        if part:
            a.set_partition(*part)
            b.set_partition(*part)
        assert np.array_equal(a.place_gangs(req, off), b.place_gangs(req, off))
        assert np.array_equal(a.read_occupancy(), b.read_occupancy())
        a.close()
        b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_gangs_of_one(policy):
    """F4 (d): gangs of one give a GANG_ONE_NODE engine's answer, and under first-fit and right-to-left isl_place_batch's."""
    rng = SplitMix64(6077 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 12) for _ in range(300)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, G, len(rows), 3000, 1)
    off = np.arange(len(req) + 1)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=E.FLAG_GANG_ONE_NODE)
    got = a.place_gangs(req, off)
    assert np.array_equal(got, b.place_gangs(req, off)) and np.array_equal(a.read_occupancy(), b.read_occupancy())
    if policy in (E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT):
        c = engine(node_off, rows, occ, policy, flags=0)
        assert np.array_equal(got, c.place_batch(req)) and np.array_equal(a.read_occupancy(), c.read_occupancy())
        c.close()
    a.close()
    b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_place_batch_unchanged(policy):
    """F6: every other call on a flagged engine returns what it returns on an unflagged one."""
    rng = SplitMix64(7005 + policy)
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


def test_refusals_and_states():
    """F6: isl_create refuses the flag with the other two gang flags, ISL_FLAG_ALL_NODES or node scoring; isl_place_gangs keeps its codes
    in every state."""
    lib = E.load_library()
    for policy, flags in ((E.POLICY_FIRST_FIT, FEW | E.FLAG_GANG_ONE_NODE), (E.POLICY_FIRST_FIT, FEW | E.FLAG_GANG_DISTINCT_NODES),
                          (E.POLICY_FIRST_FIT, FEW | E.FLAG_ALL_NODES), (E.POLICY_MOST_ALLOCATED, FEW), (E.POLICY_LEAST_ALLOCATED, FEW)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == E.EINVAL, (policy, flags)
    rows = E.make_profiles(tables.A100_40GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(req), p(out))

    fresh = E.Engine(max_gpus=16, max_batch=16, flags=FEW)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no profiles
    fresh.load_profiles(rows)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no inventory
    eng = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), max_batch=3)
    assert call(eng, [0, 4]) == E.ERANGE
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL
    assert call(eng, [1, 3]) == E.EINVAL
    assert lib.isl_place_gangs(eng._h, 1, None, p(req), p(out)) == E.EINVAL
    assert call(eng, [0]) == E.OK
    eng.set_partition(1, 1)
    assert call(eng, [0, 1]) == E.ERANGE                         # an empty partition
    eng = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8))
    eng.stream_open(1)
    try:
        assert call(eng, [0, 1]) == E.ESTATE                     # an open stream owns the engine
    finally:
        eng.stream_close()
    assert call(eng, [0, 2]) == E.OK
    big = engine(node_offsets(1, (1 << 20) + 8), rows, np.zeros((1 << 20) + 8, dtype=np.uint8))
    assert call(big, [0, 1]) == E.ERANGE                         # a partition of more than 2^20 GPUs
    big.set_partition(8, (1 << 20) + 8)
    assert call(big, [0, 2]) == E.OK and out["gpu"][:2].tolist() == [8, 8]
    big.close()
    fresh.close()


def test_stats_count_committed_members():
    """Members of a split gang count once it commits; those of a gang that aborts after a placed round do not."""
    rows = E.make_profiles(tables.A100_40GB)
    eng = engine(node_offsets(2, 1), rows, np.array([0x7E, 0x7E], dtype=np.uint8))
    eng.reset_stats()
    got = eng.place_gangs(alloc_requests(np.array([0, 0, 0, 0, 0], dtype=np.uint8)), [0, 3, 5])
    assert records(got) == [(E.GPU_NONE, 9, 1, E.ST_GANG_ABORTED)] * 2 + [(E.GPU_NONE, 9, 1, E.ST_NO_CAPACITY)] + \
        [(0, 0, 1, E.ST_PLACED), (1, 0, 1, E.ST_PLACED)]
    assert eng.stats()["placed"] == 2
    assert eng.read_occupancy().tolist() == [0x7F, 0x7F]


def cr_cluster(gpus_per_node):
    items = []
    for n, k in enumerate(gpus_per_node):
        spec = {"MigGPUUUID": {"GPU-%d-%d" % (n, g): "x" for g in range(k)}, "allocations": {}, "prepared": {},
                "migplacement": tables.migplacement(tables.A100_40GB)}
        items.append({"metadata": {"name": "node-%d" % n}, "spec": spec})
    return items


def pods(names, tag):
    return [{"uid": "%s%d" % (tag, i), "name": "p", "namespace": "default", "profile": name} for i, name in enumerate(names)]


def test_place_pending_gangs_few_nodes():
    """Nodes of one, one and two GPUs: the first [3g.20gb x 2] goes to node 2 whole; the second splits over nodes 0 and 1, where a
    one-node engine would leave it pending; a third gang finds no room and commits nothing."""
    items = cr_cluster([1, 1, 2])
    r = ctl.InstasliceReconciler(items, gang_few_nodes=True)
    out = r.place_pending_gangs([pods(["3g.20gb", "3g.20gb"], "a"), pods(["3g.20gb", "3g.20gb"], "b"),
                                 pods(["3g.20gb", "3g.20gb", "3g.20gb"], "c")])
    assert [v for v, _ in out] == ["placed", "placed", "none"]
    assert [a["nodename"] for a in out[0][1]] == ["node-2", "node-2"]
    assert [a["nodename"] for a in out[1][1]] == ["node-0", "node-1"]
    assert sorted(items[2]["spec"]["allocations"]) == ["a0", "a1"] and sorted(items[0]["spec"]["allocations"]) == ["b0"]
    assert np.array_equal(r.engine.read_occupancy(), GO.cr_occupancy(items))


def test_host_mirror_gang_few_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_few_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_few_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
