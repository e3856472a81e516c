"""All-or-nothing gangs (isl_place_gangs) on the H100: k_bestfit's gang instantiation against the CPU restatement of
tests/gang_oracle.py, records and final occupancy byte-identical."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle
from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_oracle as GO
from gang_oracle import KAT_OCC, KAT_RECORDS, kat_call

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=0):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if rows.ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def test_kat():
    rows = E.make_profiles(tables.A100_40GB)
    req, off = kat_call()
    eng = engine(node_offsets(1, 1), rows, np.zeros(1, dtype=np.uint8))
    for i, (a, b) in enumerate(zip(off[:-1], off[1:])):
        got = eng.place_gangs(req[a:b], [0, b - a])
        assert [tuple(int(x) for x in r) for r in got] == KAT_RECORDS[i], i
        assert int(eng.read_occupancy()[0]) == KAT_OCC[i], i
    eng.load_inventory(node_offsets(1, 1), np.zeros(1, dtype=np.uint8))
    got = eng.place_gangs(req, off)
    assert [tuple(int(x) for x in r) for r in got] == [r for g in KAT_RECORDS for r in g]
    assert int(eng.read_occupancy()[0]) == KAT_OCC[-1]


def test_gang_spans_two_nodes():
    rows = E.make_profiles(tables.A100_40GB)
    eng = engine(node_offsets(2, 1), rows, np.zeros(2, dtype=np.uint8))
    got = eng.place_gangs(alloc_requests(np.array([2, 2], dtype=np.uint8)), [0, 2])
    assert [tuple(int(x) for x in r) for r in got] == [(0, 0, 4, E.ST_PLACED), (1, 0, 4, E.ST_PLACED)]
    assert eng.read_occupancy().tolist() == [0x0F, 0x0F]


def gang_mix(rng, kind, n):
    if kind == "ones":
        return np.arange(n + 1, dtype=np.uint32)
    if kind == "whole":
        return np.array([0, n], dtype=np.uint32)
    off = [0]
    if kind == "straddle":          # small gangs around one gang of 33..100 members that crosses 32-request blocks
        big_at = 5 + int(rng.next1() % 20)
        off.append(big_at)
        off.append(big_at + 33 + int(rng.next1() % 68))
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % 40)))
    return np.asarray(off, dtype=np.uint32)


def random_call(rng, G, n_names, n):
    """ALLOCs of every profile (a few unknown ones), FREEs (a few malformed) and NOOPs scattered through the gangs."""
    req = alloc_requests((rng.next(n) % np.uint64(n_names + 1)).astype(np.uint8))
    req["profile"][req["profile"] == n_names] = E.PROFILE_UNKNOWN
    for i in np.flatnonzero(rng.next(n) % np.uint64(11) == 0):
        g = int(rng.next1() % (G + 2))              # G, G + 1: BAD_SPAN
        start = int(rng.next1() % 8)
        req[i] = (g, 0, E.OP_FREE, start, 1 + int(rng.next1() % (8 - start)))
    req["op"][rng.next(n) % np.uint64(29) == 0] = E.OP_NOOP
    return req


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
@pytest.mark.parametrize("G", [1000, 4608])
def test_vs_oracle(policy, quirks, n_tables, G):
    """G on both sides of kBfSmemGpus (class bitmaps in shared or global memory), one table or three per-node tables, gangs of one,
    of 1..40, one gang straddling 32-request blocks, and one gang that is the whole call."""
    rng = SplitMix64(policy * 1000 + quirks * 100 + n_tables * 10 + G)
    n_nodes = G // 8
    node_off = node_offsets(n_nodes, 8)
    if n_tables == 1:
        rows, node_table = E.make_profiles(tables.H100_80GB), None
        n_names = len(rows)
        sizes = GO.default_sizes(rows)
    else:
        names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
        node_table = (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8)
        n_names = len(names)
        sizes = GO.default_sizes(rows, node_table)
    n = 300 if policy == E.POLICY_MIN_FRAG else 2500
    outcomes = set()
    for kind in ("ones", "mixed", "straddle", "whole"):
        occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)   # dense: profiles run out and gangs abort
        req = random_call(rng, G, n_names, n)
        off = gang_mix(rng, kind, n)
        ref = oracle.Fast(node_off, rows, quirks, policy, node_table=node_table)
        ref.load(occ)
        want = GO.fast_place_gangs(ref, req, off, sizes)
        eng = engine(node_off, rows, occ, policy, quirks, node_table)
        got = eng.place_gangs(req, off)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (kind, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
        assert np.array_equal(eng.read_occupancy(), ref.occupancy()), kind
        outcomes |= set(np.unique(got["status"]).tolist())
        eng.close()
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_FREED, E.ST_NOOP} <= outcomes


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("G", [1000, 4608])
def test_gangs_of_one_equal_place_batch(policy, G):
    """All-size-1 calls are byte-identical to isl_place_batch on a second engine with the same policy (records and occupancy)."""
    rng = SplitMix64(77 + policy + G)
    node_off = node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy)
    for _ in range(2):
        req = random_call(rng, G, len(rows), 3000 if policy != E.POLICY_MIN_FRAG else 1000)
        got, want = a.place_gangs(req, np.arange(len(req) + 1)), b.place_batch(req)
        assert np.array_equal(got, want)
        assert np.array_equal(a.read_occupancy(), b.read_occupancy())


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_partition(policy):
    """An engine restricted with isl_set_partition places gangs only inside its range; the rest of the inventory is untouched."""
    rng = SplitMix64(9)
    G, lo, hi = 256, 64, 160
    node_off = node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy)
    a.set_partition(lo, hi)
    b.set_partition(lo, hi)
    req = alloc_requests((rng.next(800) % np.uint64(len(rows))).astype(np.uint8))
    got = a.place_gangs(req, np.arange(len(req) + 1))
    assert np.array_equal(got, b.place_batch(req))
    a.load_inventory(node_off, occ)
    a.set_partition(lo, hi)
    got = a.place_gangs(req, gang_mix(rng, "mixed", len(req)))
    placed = got[got["status"] == E.ST_PLACED]
    assert len(placed) and ((placed["gpu"] >= lo) & (placed["gpu"] < hi)).all()
    after = a.read_occupancy()
    assert np.array_equal(np.r_[after[:lo], after[hi:]], np.r_[occ[:lo], occ[hi:]])


def test_error_returns():
    lib = E.load_library()
    rows = E.make_profiles(tables.A100_40GB)
    node_off, occ = node_offsets(1, 2), np.zeros(2, dtype=np.uint8)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(req), p(out))

    fresh = E.Engine(max_gpus=16, max_batch=16)
    assert call(fresh, [0, 4]) == E.ESTATE                        # no profiles or inventory
    eng = engine(node_off, rows, occ, max_batch=3)
    assert call(eng, [0, 4]) == E.ERANGE                          # more requests than max_batch
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL                    # an empty gang
    assert call(eng, [1, 3]) == E.EINVAL                          # gang_off[0] != 0
    assert lib.isl_place_gangs(eng._h, 1, None, p(req), p(out)) == E.EINVAL
    assert call(eng, [0]) == E.OK                                 # no gang at all
    eng = engine(node_off, rows, occ, flags=E.FLAG_ALL_NODES)
    assert call(eng, [0, 1]) == E.EINVAL
    eng = engine(node_off, rows, occ)
    eng.stream_open(1)
    try:
        assert call(eng, [0, 1]) == E.ESTATE                      # an open stream owns the engine
    finally:
        eng.stream_close()
    assert call(eng, [0, 1]) == E.OK


def test_stats_count_committed_members():
    rows = E.make_profiles(tables.A100_40GB)
    req, off = kat_call()
    eng = engine(node_offsets(1, 1), rows, np.zeros(1, dtype=np.uint8))
    eng.reset_stats()
    got = eng.place_gangs(req, off)
    assert eng.stats()["placed"] == int((got["status"] == E.ST_PLACED).sum()) == 4


def cluster(n_nodes, gpus):
    items = []
    for n in range(n_nodes):
        spec = {"MigGPUUUID": {"GPU-%d-%d" % (n, g): "x" for g in range(gpus)}, "allocations": {}, "prepared": {},
                "migplacement": tables.migplacement(tables.A100_40GB)}
        items.append({"metadata": {"name": "node-%d" % n}, "spec": spec})
    return items


def pods(names, tag):
    return [{"uid": "%s%d" % (tag, i), "name": "p", "namespace": "default", "profile": name} for i, name in enumerate(names)]


def test_place_pending_gangs_end_to_end():
    items = cluster(1, 1)
    r = ctl.InstasliceReconciler(items)
    gangs = [pods(["3g.20gb", "3g.20gb"], "a"), pods(["3g.20gb", "1g.5gb"], "b"), pods(["1g.5gb", "2g.10gb"], "c"),
             pods(["1g.5gb", "1g.5gb"], "d"), pods(["1g.5gb"], "e")]
    out = r.place_pending_gangs(gangs)
    assert [v for v, _ in out] == ["none", "placed", "none", "placed", "none"]
    assert [(a["start"], a["size"], a["podUUID"]) for a in out[1][1]] == [(0, 4, "b0"), (4, 1, "b1")]
    assert sorted(items[0]["spec"]["allocations"]) == ["b0", "b1", "d0", "d1"]      # placed gangs only
    assert int(GO.cr_occupancy(items)[0]) == int(r.engine.read_occupancy()[0]) == 0x7F


def test_place_pending_gangs_veto_and_orphan_fallback():
    """A realised slice whose allocation is gone (an orphan) can veto one member: the whole gang is released, and with orphans
    present every gang is resolved on its own, so the next gang sees no trace of it."""
    items = cluster(2, 1)
    items[0]["spec"]["prepared"]["MIG-x"] = {"profile": "1g.5gb", "start": 1, "size": 1, "parent": "GPU-0-0", "podUUID": "gone",
                                             "giinfo": 0, "ciinfo": 0}
    r = ctl.InstasliceReconciler(items)
    out = r.place_pending_gangs([pods(["1g.5gb", "1g.5gb"], "a"), pods(["2g.10gb", "1g.5gb", "3g.20gb"], "b")])
    assert [v for v, _ in out] == ["veto", "placed"]
    assert [(a["gpuUUID"], a["start"]) for a in out[1][1]] == [("GPU-0-0", 0), ("GPU-0-0", 2), ("GPU-1-0", 0)]
    assert sorted(k for it in items for k in it["spec"]["allocations"]) == ["b0", "b1", "b2"]
    assert np.array_equal(r.engine.read_occupancy(), GO.cr_occupancy(items))


def test_host_mirror_gangs_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gangs_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gangs_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
