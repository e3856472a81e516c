"""One-node gangs (isl_place_gangs on an engine created with ISL_FLAG_GANG_ONE_NODE) on the H100: k_ganglocal<one_node> against the brute
force of tests/gang_node_fast.cpp, records and final occupancy byte-identical, plus the hand-worked vectors, the identities and refusals of
include/islplace.h (G1-G6), the reconciler flow and the C++ host mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_node_fast as GNF
import gang_node_oracle as GNO
import gang_oracle as GO

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
ONE_NODE = E.FLAG_GANG_ONE_NODE


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=ONE_NODE):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
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


def assert_gangs_on_one_node(eng, got, off):
    """Every committed gang's PLACED members are on one node (isl_gpu_to_node)."""
    for a, b in zip(off[:-1], off[1:]):
        placed = got[a:b][got[a:b]["status"] == E.ST_PLACED]
        assert len({eng.gpu_to_node(int(g)) for g in placed["gpu"]}) <= 1, (a, b)


@pytest.mark.parametrize("kat", list(GNO.load_kat()), ids=lambda k: k[0])
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


def random_call(rng, G, n_names, n, max_gang):
    req = alloc_requests((rng.next(n) % np.uint64(n_names + 1)).astype(np.uint8))
    req["profile"][req["profile"] == n_names] = E.PROFILE_UNKNOWN
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


def check(node_off, rows, occ, node_table, req, off, policy, quirks, part=None, max_batch=1 << 16):
    G = int(node_off[-1])
    lo, hi = part or (0, G)
    want, occ_want = GNF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
    eng = engine(node_off, rows, occ, policy, quirks, node_table, max_batch=max_batch)
    if part:
        eng.set_partition(lo, hi)
    got = eng.place_gangs(req, off)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want)
    assert_gangs_on_one_node(eng, got, off)
    eng.close()
    return got


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_vs_brute_force(policy, quirks, n_tables):
    """Nodes of 1 to 16 GPUs with empty nodes among them, gangs of 1..12 with FREEs, NOOPs and unknown profiles, whole and cut."""
    rng = SplitMix64(policy * 100 + quirks * 10 + n_tables)
    outcomes = set()
    for trial in range(4):
        sizes = [int(rng.next1() % 17) for _ in range(150)]
        node_off, rows, occ, node_table, n_names = cluster(rng, n_tables, sizes, 0x3F if trial % 2 else 0x7F)
        G = int(node_off[-1])
        req, off = random_call(rng, G, n_names, 600 if policy == E.POLICY_MIN_FRAG else 1500, 12)
        part = None if trial < 2 else (int(rng.next1() % (G // 3)), G - int(rng.next1() % (G // 3)))
        got = check(node_off, rows, occ, node_table, req, off, policy, quirks, part)
        outcomes |= set(np.unique(got["status"]).tolist())
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_FREED, E.ST_NOOP} <= outcomes


@pytest.mark.parametrize("shape", [(1, 1), (1, 4096), (3, 4096), (4096, 1), (1024, 8), (131072, 8), (1 << 20, 1), (1, 1 << 20)],
                         ids=lambda s: "%dx%d" % s)
@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_scale(shape, policy):
    """Inventories from one GPU to 2^20 GPUs (2^20 nodes of one), nodes of up to 4096 GPUs, and one node of 2^20 GPUs, which one CTA
    owns: its share does not fit in shared memory and lives in global memory; gangs up to max_batch members."""
    n_nodes, per = shape
    G = n_nodes * per
    rng = SplitMix64(G + policy)
    node_off = node_offsets(n_nodes, per)
    rows = E.make_profiles(tables.H100_80GB)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    n = 64 if G > 65536 else 256
    req, off = random_call(rng, G, len(rows), n, 24)
    check(node_off, rows, occ, None, req, off, policy, E.QUIRKS_REF_EXACT, max_batch=n)
    whole = np.array([0, n], dtype=np.uint32)           # one gang of max_batch members
    check(node_off, rows, occ, None, req, whole, policy, E.QUIRKS_REF_EXACT, max_batch=n)


def test_share_in_global_memory_uneven():
    """Three CTAs of which one owns a node of 2^20 - 8 GPUs and two own tiny nodes: the shares live in global memory."""
    G = 1 << 20
    rng = SplitMix64(4242)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.array([0, 5, G - 3, G], dtype=np.uint32)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 48, 6)
    for policy in POLICIES:
        check(node_off, rows, occ, None, req, off, policy, E.QUIRKS_REF_EXACT, max_batch=48)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_one_node_equals_unflagged(policy, quirks):
    """G4: a one-node inventory, and a partition inside one node of a larger inventory, give the unflagged engine's answer."""
    rng = SplitMix64(40 + policy * 3 + quirks)
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


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_gangs_of_one_equal_place_batch(policy):
    """G4: gangs of one on a flagged first-fit or right-to-left engine are isl_place_batch."""
    rng = SplitMix64(77 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 12) for _ in range(300)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, G, len(rows), 3000, 1)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=0)
    assert np.array_equal(a.place_gangs(req, np.arange(len(req) + 1)), b.place_batch(req))
    assert np.array_equal(a.read_occupancy(), b.read_occupancy())


@pytest.mark.parametrize("policy", POLICIES)
def test_place_batch_unchanged(policy):
    """G5: every other call on a flagged engine returns what it returns on an unflagged one."""
    rng = SplitMix64(5 + policy)
    node_off = node_offsets(500, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(4000) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, 4000, len(rows), 5000, 1)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, flags=0)
    assert np.array_equal(a.place_batch(req), b.place_batch(req))
    assert np.array_equal(a.place_batch_range(800, 1600, req), b.place_batch_range(800, 1600, req))
    assert np.array_equal(a.read_occupancy(), b.read_occupancy())


def test_refusals_and_states():
    """G5: isl_create refuses the flag with ISL_FLAG_ALL_NODES or node scoring; isl_place_gangs keeps its codes in every state."""
    lib = E.load_library()
    for policy, flags in ((E.POLICY_FIRST_FIT, ONE_NODE | E.FLAG_ALL_NODES), (E.POLICY_MOST_ALLOCATED, ONE_NODE),
                          (E.POLICY_LEAST_ALLOCATED, ONE_NODE)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == E.EINVAL
    rows = E.make_profiles(tables.A100_40GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(req), p(out))

    fresh = E.Engine(max_gpus=16, max_batch=16, flags=ONE_NODE)
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


def test_stats_count_committed_members():
    rows = E.make_profiles(tables.A100_40GB)
    eng = engine(node_offsets(2, 1), rows, np.zeros(2, dtype=np.uint8))
    eng.reset_stats()
    got = eng.place_gangs(alloc_requests(np.array([2, 2, 0, 0, 2], dtype=np.uint8)), [0, 2, 4, 5])
    assert records(got)[2:] == [(0, 0, 1, E.ST_PLACED), (0, 1, 1, E.ST_PLACED), (1, 0, 4, E.ST_PLACED)]
    assert eng.stats()["placed"] == 3


def cr_cluster(gpus_per_node):
    items = []
    for n, k in enumerate(gpus_per_node):
        spec = {"MigGPUUUID": {"GPU-%d-%d" % (n, g): "x" for g in range(k)}, "allocations": {}, "prepared": {},
                "migplacement": tables.migplacement(tables.A100_40GB)}
        items.append({"metadata": {"name": "node-%d" % n}, "spec": spec})
    return items


def pods(names, tag):
    return [{"uid": "%s%d" % (tag, i), "name": "p", "namespace": "default", "profile": name} for i, name in enumerate(names)]


def test_place_pending_gangs_one_node():
    items = cr_cluster([1, 1, 2])
    r = ctl.InstasliceReconciler(items, gang_one_node=True)
    out = r.place_pending_gangs([pods(["3g.20gb", "3g.20gb"], "a"), pods(["3g.20gb", "3g.20gb"], "b"), pods(["1g.5gb", "1g.5gb"], "c")])
    assert [v for v, _ in out] == ["placed", "none", "placed"]
    assert [(a["gpuUUID"], a["nodename"]) for a in out[0][1]] == [("GPU-2-0", "node-2"), ("GPU-2-1", "node-2")]
    assert [(a["gpuUUID"], a["start"]) for a in out[2][1]] == [("GPU-0-0", 0), ("GPU-0-0", 1)]
    assert sorted(items[2]["spec"]["allocations"]) == ["a0", "a1"] and sorted(items[0]["spec"]["allocations"]) == ["c0", "c1"]
    assert np.array_equal(r.engine.read_occupancy(), GO.cr_occupancy(items))
    plain = ctl.InstasliceReconciler(cr_cluster([1, 1, 2]))
    assert [a["nodename"] for a in plain.place_pending_gangs([pods(["3g.20gb", "3g.20gb"], "a")])[0][1]] == ["node-0", "node-1"]


def test_host_mirror_gang_node_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_node_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_node_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
