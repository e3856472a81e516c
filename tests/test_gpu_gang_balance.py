"""Balanced gangs (isl_place_gangs on an engine created with ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_BALANCED) on the H100:
k_ganglocal<per_gang, balanced> and <per_gang, min_members, balanced> against the brute force of tests/gang_balance_fast.cpp (records,
occupancy, stats.placed) on the hand-worked vectors, random clusters with every locality byte, thousands of nodes, partitions that cut
nodes, shares on both sides of the shared-memory switch, 16 profiles, 8 node tables, 2^20 GPUs and counts past 255; B4 device against
device; elastic trims; B6 and the codes of every engine state; the reconciler and the C++ mirror."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_balance_fast as GBF
import gang_balance_oracle as GBO
import gang_locality_oracle as GLO
from test_gang_balance_oracle import random_bytes, random_minima
from test_gang_spread_oracle import random_cluster, random_gangs
from test_gpu_gang_few import cr_cluster, device, pods, random_call
from test_oracle_gang_topology_limits import CASES, FIXTURES, LAYOUT_CASES, case_ids, gang_plan, layout_cases, small_gangs
from test_oracle_request_major_limits import gang_call, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
BAL = E.FLAG_GANG_LOCALITY | E.FLAG_GANG_BALANCED


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, flags=BAL, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16):
    eng = E.Engine(max_gpus=max(4097, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if np.asarray(rows).ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def check(node_off, rows, occ, req, off, quirks, policy, node_table=None, lo=0, hi=None, elastic=False, what=""):
    """One call on a flagged engine against the brute force: records, occupancy and stats.placed."""
    G = int(node_off[-1])
    hi = G if hi is None else hi
    eng = engine(node_off, rows, occ, policy, BAL | (E.FLAG_GANG_MIN_MEMBERS if elastic else 0), quirks, node_table,
                 max_batch=max(16, len(req)))
    if (lo, hi) != (0, G):
        eng.set_partition(lo, hi)
    want, occ_want, placed = GBF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, elastic=elastic)
    eng.reset_stats()
    got = eng.place_gangs(req, off)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    assert eng.stats()["placed"] == placed, what
    eng.close()
    return got


@pytest.mark.parametrize("kat", list(GBO.load_kat()), ids=lambda k: k[0])
def test_kat(kat):
    _name, inputs, req, off, want, occ_after, placed = kat
    lo, hi = inputs["partition"] or (0, int(inputs["node_off"][-1]))
    got = check(inputs["node_off"], inputs["rows"], inputs["occ"], req, off, inputs["quirks"], inputs["policy"], inputs["node_table"], lo,
                hi, inputs["elastic"], _name)
    assert [tuple(int(x) for x in r) for r in got] == want


@pytest.mark.parametrize("elastic", [False, True])
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("policy", POLICIES)
def test_vs_brute_force(policy, quirks, elastic):
    """The CPU tests' random clusters: one or three node tables, partitions that cut nodes, FREEs, NOOPs, unknown profiles and every
    locality byte in one call."""
    rng = SplitMix64(5100 + 10 * policy + 3 * quirks + 100 * elastic)
    for trial in range(16):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 1 + 2 * (trial % 2))
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 4 < 2 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 60, max_gang=8)
        req = GLO.with_locality(req, off, random_bytes(rng, len(off) - 1))
        if elastic:
            req = random_minima(rng, req, off)
        check(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, elastic, trial)


@pytest.mark.parametrize("policy", POLICIES)
def test_large_vs_brute_force(policy):
    """Thousands of GPUs in nodes of 1-16 with three node tables: many CTAs, gangs of up to 24, partitions cutting nodes."""
    rng = SplitMix64(5200 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 16) for _ in range(700)]).astype(np.uint32)
    G = int(node_off[-1])
    _, rows = E.make_profile_tables([tables.H100_80GB, tables.A30_24GB, tables.A100_40GB])
    node_table = (rng.next(700) % np.uint64(3)).astype(np.uint8)
    occ = (rng.next(G) & np.uint64(0x7B)).astype(np.uint8)
    req, off = random_call(rng, G, rows.shape[1], 4000, 24)
    req = GLO.with_locality(req, off, random_bytes(rng, len(off) - 1))
    for part in ((0, G), (int(rng.next1() % 100) + 3, G - 50)):
        check(node_off, rows, occ, req, off, E.QUIRKS_FIXED, policy, node_table, *part, what=part)


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_edges(case):
    """Every edge of the CTA layout built from this device's SM count and the balanced instantiations' own shared-memory opt-in (their
    256 B of static shared memory), shares on both sides of the shared / global memory switch among them, 8 node tables."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    assert edge(gang_plan(node_off, lo, hi, sms, optin - 256)), case
    i = LAYOUT_CASES.index(case)
    rows = t8tab()
    rng = SplitMix64(5300 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    off = small_gangs(rng, 400, 8)
    req = GLO.with_locality(gang_call(rng, G, 16, 400), off, random_bytes(rng, len(off) - 1))
    check(node_off, rows, whole_bytes(rng, G, dense=True), req, off, E.QUIRKS_FIXED, POLICIES[i % 4], node_table, lo, hi, i % 2 == 1,
          case)


@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_table_limits(name, quirks):
    """16 profiles and 8 node tables: every fixture of the table-limit suite."""
    rows = FIXTURES[name]()
    rng = SplitMix64(5400 + CASES.index((name, quirks)))
    n_nodes = 300
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 8) for _ in range(n_nodes)]).astype(np.uint32)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes) if np.asarray(rows).ndim == 2 else None
    n_names = np.asarray(rows).shape[-1]
    off = small_gangs(rng, 800, 8)
    req = GLO.with_locality(gang_call(rng, G, n_names, 800), off, random_bytes(rng, len(off) - 1))
    check(node_off, rows, whole_bytes(rng, G), req, off, quirks, POLICIES[CASES.index((name, quirks)) % 4], node_table, what=name)


@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy):
    """A 2^20-GPU partition of 8-GPU nodes (the cap), balanced gangs of replicas at maxSkew 1 and 2 among the other localities."""
    rng = SplitMix64(5500 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.arange(0, (1 << 20) + 1, 8, dtype=np.uint32)
    G = int(node_off[-1])
    occ = whole_bytes(rng, G, dense=True)
    req, off = random_call(rng, G, len(rows), 300, 24)
    req = GLO.with_locality(req, off, random_bytes(rng, len(off) - 1))
    got = check(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy, what=policy)
    assert (got["status"] == E.ST_PLACED).any()


@pytest.mark.parametrize("policy", POLICIES)
def test_counts_past_255(policy):
    """Two 64-GPU nodes and a one-GPU node take a gang of 900 1g.10gb: the counts of the big nodes reach 448, and the choice at every
    member depends on them being exact; at maxSkew 1, 2 and 200, and a gang one member too large."""
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.array([0, 64, 128, 129], dtype=np.uint32)
    occ = np.zeros(129, dtype=np.uint8)
    for skew in (1, 2, 200):
        for n in (900, 904):
            req = GLO.with_locality(alloc_requests(np.zeros(n, dtype=np.uint8)), [0, n], [E.gang_balanced_nodes(skew)])
            got = check(node_off, rows, occ, req, [0, n], E.QUIRKS_REF_EXACT, policy, what=(skew, n))
            assert (got["status"] == E.ST_PLACED).all() == (n == 900)
            if n == 900 and skew == 1:
                counts = np.bincount(np.searchsorted(node_off, got["gpu"].astype(np.int64), side="right") - 1, minlength=3)
                assert sorted(counts.tolist()) == [7, 446, 447], counts


@pytest.mark.parametrize("policy", POLICIES)
def test_b4_device(policy):
    """B4 device against device: (a) committed distinct-node gangs equal byte 4; (b) a skew of at least the gang equals byte 0; (c) a
    partition inside one node equals byte 0; (d) gangs of one equal byte 0, and isl_place_batch under FIRST_FIT and RIGHT_TO_LEFT;
    (e) a call mixing every locality equals its gangs one at a time."""
    rng = SplitMix64(5600 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 10) for _ in range(300)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
    req, off = random_call(rng, G, len(rows), 1500, 8)
    n_gangs = len(off) - 1
    k = np.add.reduceat((req["op"] == E.OP_ALLOC).astype(np.int64), off[:-1].astype(np.int64))

    def run(r, o=off, part=None, flags=BAL):
        eng = engine(node_off, rows, occ, policy, flags)
        if part:
            eng.set_partition(*part)
        eng.reset_stats()
        got = eng.place_gangs(r, o)
        res = (got, eng.read_occupancy(), eng.stats()["placed"])
        eng.close()
        return res

    def same(a, b):
        return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]

    # (a) each gang alone on the same occupancy: where byte 3 commits, byte 4 gives the same records
    seen = 0
    eng = engine(node_off, rows, occ, policy)
    for a, b in zip(off[:-1], off[1:]):
        alloc = req["op"][a:b] == E.OP_ALLOC
        if not alloc.any() or (req["op"][a:b] == E.OP_FREE).any():
            continue
        eng.load_inventory(node_off, occ)
        ga = eng.place_gangs(GLO.with_locality(req[a:b], [0, b - a], [3]), [0, b - a])
        if (ga["status"][alloc] == E.ST_PLACED).all():
            occ_a = eng.read_occupancy()
            eng.load_inventory(node_off, occ)
            assert np.array_equal(eng.place_gangs(GLO.with_locality(req[a:b], [0, b - a], [4]), [0, b - a]), ga)
            assert np.array_equal(eng.read_occupancy(), occ_a)
            seen += 1
        if seen == 20:
            break
    eng.close()
    assert seen > 5
    # (b)
    zero = run(req)
    assert same(run(GLO.with_locality(req, off, 3 + np.maximum(k, 1))), zero)
    # (c)
    j = int(np.argmax(np.diff(node_off)))
    part = (int(node_off[j]), int(node_off[j + 1]))
    assert same(run(GLO.with_locality(req, off, random_bytes(rng, n_gangs, True)), part=part), run(req, part=part))
    # (d)
    ones = np.arange(len(req) + 1, dtype=np.uint32)
    single = run(GLO.with_locality(req, ones, random_bytes(rng, len(req), True)), ones)
    assert same(single, run(req, ones))
    if policy in (E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT):
        eng = engine(node_off, rows, occ, policy, 0)
        eng.reset_stats()
        assert np.array_equal(single[0], eng.place_batch(req))
        assert np.array_equal(single[1], eng.read_occupancy()) and single[2] == eng.stats()["placed"]
        eng.close()
    # (e)
    mixed = GLO.with_locality(req, off, random_bytes(rng, n_gangs))
    whole = run(mixed)
    eng = engine(node_off, rows, occ, policy)
    alloc = mixed["op"] == E.OP_ALLOC
    frees = mixed.copy()
    frees["op"][alloc] = E.OP_NOOP
    eng.reset_stats()
    out = eng.place_gangs(frees, [0, len(req)])
    for a, b in zip(off[:-1], off[1:]):
        if alloc[a:b].any():
            members = mixed[a:b].copy()
            members["op"][~alloc[a:b]] = E.OP_NOOP
            out[a:b][alloc[a:b]] = eng.place_gangs(members, [0, b - a])[alloc[a:b]]
    assert np.array_equal(out, whole[0]) and np.array_equal(eng.read_occupancy(), whole[1]) and eng.stats()["placed"] == whole[2]
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_elastic_trims(policy):
    """B5: replicas at maxSkew 1 and 2 on a cluster with less room than the gangs; the leading run commits when it reaches the minimum."""
    rng = SplitMix64(5700 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = node_offsets(40, 2)
    occ = np.where(rng.next(80) % np.uint64(2) == 0, 0x7F, 0x1F).astype(np.uint8)
    sizes = [30, 12, 25, 40, 8]
    off = np.cumsum([0] + sizes).astype(np.uint32)
    req = alloc_requests(np.zeros(int(off[-1]), dtype=np.uint8))
    req = GLO.with_locality(req, off, [4, 5, 4, 5, 3])
    per = np.repeat(np.array([20, 0, 10, 1, 2]), sizes)
    req["size"] = per
    got = check(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy, elastic=True, what=policy)
    assert (got["status"] == E.ST_GANG_TRIMMED).any() and (got["status"] == E.ST_PLACED).any()


def test_refusals_and_states():
    """B6: isl_create's refusals and acceptances; B1 and L4: a byte above 3 without the flag, or two bytes in one gang, is EINVAL before
    the state and changes nothing; isl_place_gangs keeps its codes in every state (no profiles, no inventory, a snapshot, an open stream,
    more than max_batch, an empty and a 2^20 + 8 GPU partition); isl_preempt keeps P1's refusal of a balanced byte; the binding refuses
    bytes beyond 255 on a flagged engine."""
    lib = E.load_library()
    for policy, flags, rc in ((E.POLICY_FIRST_FIT, E.FLAG_GANG_BALANCED, E.EINVAL), (E.POLICY_MOST_ALLOCATED, BAL, E.EINVAL),
                              (E.POLICY_LEAST_ALLOCATED, BAL | E.FLAG_GANG_NODE_SCORE, E.EINVAL), (E.POLICY_FIRST_FIT, BAL | E.FLAG_ALL_NODES, E.EINVAL),
                              (E.POLICY_BEST_FIT, E.FLAG_GANG_BALANCED | E.FLAG_GANG_DISTINCT_NODES, E.EINVAL),
                              (E.POLICY_FIRST_FIT, BAL, E.OK), (E.POLICY_MIN_FRAG, BAL | E.FLAG_GANG_MIN_MEMBERS, E.OK),
                              (E.POLICY_RIGHT_TO_LEFT, BAL | E.FLAG_GANG_PREEMPT, E.OK)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == rc, (policy, flags)
        if rc == E.OK:
            lib.isl_destroy(h)
    rows = E.make_profiles(tables.A100_40GB)
    req = GLO.with_locality(alloc_requests(np.zeros(4, dtype=np.uint8)), [0, 4], [E.gang_balanced_nodes(1)])
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off, r=req):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(r), p(out))

    fresh = E.Engine(max_gpus=16, max_batch=16, flags=BAL)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no profiles
    fresh.load_profiles(rows)
    assert call(fresh, [0, 1]) == E.ESTATE                       # no inventory
    mixed = req.copy()
    mixed["start"][1] = 5
    assert call(fresh, [0, 2], mixed) == E.EINVAL                # L4 before the state
    unflagged = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), flags=E.FLAG_GANG_LOCALITY)
    assert call(unflagged, [0, 2]) == E.EINVAL                   # B1: without the flag a byte above 3 is refused
    unflagged.close()
    eng = engine(node_offsets(2, 2), rows, np.array([0x01, 0, 0, 0], dtype=np.uint8), max_batch=3)
    eng.snapshot_occupancy()
    before = (eng.read_occupancy().tolist(), eng.stats())
    assert call(eng, [0, 4]) == E.ERANGE
    assert call(eng, [0, 2], mixed) == E.EINVAL
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL
    assert lib.isl_place_gangs(eng._h, 1, None, p(req), p(out)) == E.EINVAL
    assert (eng.read_occupancy().tolist(), eng.stats()) == before
    with pytest.raises(ValueError):
        eng.place_gangs(req[:2], [0, 2], [256])
    with pytest.raises(ValueError):
        E.gang_balanced_nodes(253)
    assert eng.restore_occupancy() is None                       # the snapshot is still there
    assert call(eng, [0, 3], req[:3]) == E.OK
    assert [(int(r["gpu"]), int(r["start"])) for r in out[:3]] == [(0, 1), (2, 0), (0, 2)]
    eng.set_partition(1, 1)
    assert call(eng, [0, 1]) == E.ERANGE                         # an empty partition
    eng.close()
    eng = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8))
    eng.stream_open(1)
    try:
        assert call(eng, [0, 1]) == E.ESTATE                     # an open stream owns the engine
    finally:
        eng.stream_close()
    assert call(eng, [0, 4]) == E.OK and out["gpu"][:4].tolist() == [0, 2, 0, 2]
    eng.close()
    pre = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), flags=BAL | E.FLAG_GANG_PREEMPT)
    with pytest.raises(E.EngineError):                           # P1: isl_preempt refuses a balanced byte
        pre.preempt(req[:2], np.full(2, 5, dtype=np.uint8), np.zeros(0, dtype=E.VICTIM_DTYPE), gang_off=[0, 2],
                    locality=[E.gang_balanced_nodes(1)])
    pre.close()
    fresh.close()
    big = engine(node_offsets(1, (1 << 20) + 8), rows, np.zeros((1 << 20) + 8, dtype=np.uint8))
    assert call(big, [0, 1]) == E.ERANGE                         # a partition of more than 2^20 GPUs
    big.set_partition(8, (1 << 20) + 8)
    assert call(big, [0, 2]) == E.OK and out["gpu"][:2].tolist() == [8, 8]
    big.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_place_batch_unchanged(policy):
    """B6: every other call on a flagged engine returns what it returns on an engine without the flag."""
    rng = SplitMix64(5800 + policy)
    node_off = node_offsets(500, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(4000) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, 4000, len(rows), 5000, 1)
    a, b = engine(node_off, rows, occ, policy), engine(node_off, rows, occ, policy, E.FLAG_GANG_LOCALITY)
    assert np.array_equal(a.capacity(), b.capacity())
    assert all(np.array_equal(x, y) for x, y in zip(a.what_if(req), b.what_if(req)))
    assert np.array_equal(a.place_batch(req), b.place_batch(req))
    assert np.array_equal(a.place_batch_range(800, 1600, req), b.place_batch_range(800, 1600, req))
    assert np.array_equal(a.read_occupancy(), b.read_occupancy())
    a.close()
    b.close()


def test_place_pending_gangs_balanced():
    """Six replicas on three one-GPU nodes at maxSkew 1 land two per node; the same Deployment as a distinct-node gang stays pending."""
    items = cr_cluster([1, 1, 1])
    r = ctl.InstasliceReconciler(items, gang_locality=True, gang_balanced=True)
    out = r.place_pending_gangs([pods(["1g.5gb"] * 6, "a"), pods(["1g.5gb"] * 4, "b")],
                                locality=[E.gang_balanced_nodes(1), E.GANG_DISTINCT_NODES])
    assert [v for v, _ in out] == ["placed", "none"]
    assert [a["nodename"] for a in out[0][1]] == ["node-0", "node-1", "node-2"] * 2


def test_host_mirror_gang_balance_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_balance_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_balance_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
