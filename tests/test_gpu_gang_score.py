"""Node-scored gangs (isl_place_gangs on an engine created with ISL_FLAG_GANG_NODE_SCORE) on the H100: the node-scored k_ganglocal
instantiations against the brute force of tests/gang_score_fast.cpp (records, occupancy, stats.placed) on the CPU tests' random matrix and
the hand-worked vectors, N8 (a) device against device against k_nodefit, N8 (c) against a FIRST_FIT engine, N7 (every other entry point
as without the flag, isl_preempt as on FIRST_FIT), N1 and the codes of every engine state, the limits (2^20 GPUs, 2^20 one-GPU nodes,
shares on both sides of the shared-memory switch, 16 profiles, 8 node tables of different widths), the reconciler and the C++ mirror."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_score_fast as GSF
import gang_score_oracle as GSO
from test_gpu_gang_few import cr_cluster, device, pods, random_call
from test_oracle_gang_topology_limits import CASES, FIXTURES, LAYOUT_CASES, case_ids, gang_plan, layout_cases, small_gangs
from test_oracle_request_major_limits import gang_call, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
POLICIES = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]
SCORE = E.FLAG_GANG_NODE_SCORE
LOCALITIES = [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GSO.PER_GANG]


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


def check(inputs, what=""):
    """One call on a flagged engine against the brute force: records, occupancy and stats.placed."""
    node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, loc = inputs
    eng = engine(node_off, rows, occ, policy, SCORE | GSO.FLAGS[loc], quirks, node_table, max_batch=max(16, len(req)))
    if (lo, hi) != (0, int(node_off[-1])):
        eng.set_partition(lo, hi)
    want, occ_want, placed = GSO.run(GSF.place_gangs, inputs)
    eng.reset_stats()
    got = eng.place_gangs(req, off)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    assert eng.stats()["placed"] == placed, what
    eng.close()
    return got


@pytest.mark.parametrize("case", GSO.kat_cases(), ids=lambda c: c["name"])
def test_kat(case):
    got = check(GSO.case_inputs(case), case["name"])
    assert [tuple(int(x) for x in r) for r in got] == [tuple(w) for w in GSO.expected(case)[0]]


@pytest.mark.parametrize("locality", LOCALITIES)
@pytest.mark.parametrize("policy", POLICIES)
def test_vs_brute_force(policy, locality):
    """The CPU tests' random matrix: one to three node tables, both quirk sets, partitions, FREEs, NOOPs and unknown profiles."""
    rnd = random.Random(9100 + 10 * policy + locality)
    for i in range(40):
        _, rows = GSO.random_rows(rnd)
        check(GSO.random_case(rnd, rnd.randint(1, 40), rnd.randint(1, 24), rows, locality=locality, policy=policy), i)


@pytest.mark.parametrize("locality", LOCALITIES)
@pytest.mark.parametrize("policy", POLICIES)
def test_large_vs_brute_force(policy, locality):
    """Thousands of GPUs in nodes of 1-16 with three node tables: many CTAs, gangs of up to 8."""
    rng = SplitMix64(9200 + 10 * policy + locality)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 16) for _ in range(700)]).astype(np.uint32)
    G = int(node_off[-1])
    _, rows = E.make_profile_tables([tables.H100_80GB, tables.A30_24GB, tables.A100_40GB])
    node_table = (rng.next(700) % np.uint64(3)).astype(np.uint8)
    occ = (rng.next(G) & np.uint64(0x7B)).astype(np.uint8)
    req, off = random_call(rng, G, rows.shape[1], 4000, 8)
    if locality == GSO.PER_GANG:
        per = np.repeat(np.array([0, 1, 3])[(rng.next(len(off) - 1) % np.uint64(3)).astype(np.int64)], np.diff(off.astype(np.int64)))
        alloc = req["op"] == E.OP_ALLOC
        req["start"][alloc] = per[alloc]
    for part in ((0, G), (int(rng.next1() % 100) + 3, G - 50)):
        check((node_off, rows, node_table, occ, req, off, E.QUIRKS_FIXED, policy, *part, locality), part)


@pytest.mark.parametrize("policy", POLICIES)
def test_n8a_gangs_of_one_equal_k_nodefit(policy):
    """N8 (a), device against device: gangs of one, every locality, equal isl_place_batch (k_nodefit) on the same engine."""
    rng = SplitMix64(9300 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 12) for _ in range(400)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, G, len(rows), 3000, 1)
    for loc in LOCALITIES:
        r = req.copy()
        if loc == GSO.PER_GANG:
            r["start"][r["op"] == E.OP_ALLOC] = (rng.next(int((r["op"] == E.OP_ALLOC).sum())) % np.uint64(2)).astype(np.uint8) * 3
        eng = engine(node_off, rows, occ, policy, SCORE | GSO.FLAGS[loc])
        eng.reset_stats()
        got = eng.place_gangs(r, np.arange(len(r) + 1))
        occ_g, placed = eng.read_occupancy(), eng.stats()["placed"]
        eng.load_inventory(node_off, occ)
        eng.reset_stats()
        assert np.array_equal(got, eng.place_batch(r)), loc
        assert np.array_equal(occ_g, eng.read_occupancy()) and placed == eng.stats()["placed"], loc
        eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_n8c_one_node_equals_first_fit_engine(policy):
    """N8 (c), device against device: a partition inside one node, and a one-node inventory, equal a FIRST_FIT engine with the same
    locality flags (records and occupancy)."""
    rng = SplitMix64(9400 + policy)
    rows = E.make_profiles(tables.A100_40GB)
    for flags in (0, E.FLAG_GANG_ONE_NODE, E.FLAG_GANG_DISTINCT_NODES, E.FLAG_GANG_LOCALITY):
        for node_off, part in ((node_offsets(8, 64), (70, 120)), (np.array([0, 300], dtype=np.uint32), None)):
            G = int(node_off[-1])
            occ = (rng.next(G) & np.uint64(0x5D)).astype(np.uint8)
            req, off = random_call(rng, G, len(rows), 300, 5)
            if flags & E.FLAG_GANG_LOCALITY:
                per = np.repeat(np.array([0, 1, 3])[(rng.next(len(off) - 1) % np.uint64(3)).astype(np.int64)], np.diff(off.astype(np.int64)))
                req["start"][req["op"] == E.OP_ALLOC] = per[req["op"] == E.OP_ALLOC]
            a, b = engine(node_off, rows, occ, policy, SCORE | flags), engine(node_off, rows, occ, E.POLICY_FIRST_FIT, flags)
            if part:
                a.set_partition(*part)
                b.set_partition(*part)
            assert np.array_equal(a.place_gangs(req, off), b.place_gangs(req, off)), flags
            assert np.array_equal(a.read_occupancy(), b.read_occupancy()), flags
            a.close()
            b.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_n7_other_entry_points_unchanged(policy):
    """N7: isl_place_batch, _range, isl_what_if, isl_capacity and isl_preempt on a flagged engine return what the engine without the
    bit returns; with ISL_FLAG_GANG_PREEMPT isl_preempt returns what a FIRST_FIT engine with the same flags minus this one returns."""
    rng = SplitMix64(9500 + policy)
    node_off = node_offsets(300, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(2400) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_call(rng, 2400, len(rows), 3000, 1)
    allocs = req[req["op"] == E.OP_ALLOC][:200]
    victims = np.zeros(0, dtype=E.VICTIM_DTYPE)
    prio = np.full(len(allocs), 5, dtype=np.uint8)
    for flags in (0, E.FLAG_GANG_ONE_NODE, E.FLAG_GANG_DISTINCT_NODES, E.FLAG_GANG_LOCALITY):
        a, b = engine(node_off, rows, occ, policy, SCORE | flags), engine(node_off, rows, occ, policy, 0)
        assert np.array_equal(a.capacity(), b.capacity())
        wa, wb = a.what_if(req), b.what_if(req)
        assert all(np.array_equal(x, y) for x, y in zip(wa, wb))
        assert [np.array_equal(x, y) for x, y in zip(a.preempt(allocs, prio, victims), b.preempt(allocs, prio, victims))] == [True, True]
        assert np.array_equal(a.place_batch(req), b.place_batch(req))
        assert np.array_equal(a.place_batch_range(800, 1600, req), b.place_batch_range(800, 1600, req))
        assert np.array_equal(a.read_occupancy(), b.read_occupancy())
        a.close()
        b.close()
        pflags = flags | E.FLAG_GANG_PREEMPT
        a, c = engine(node_off, rows, occ, policy, SCORE | pflags), engine(node_off, rows, occ, E.POLICY_FIRST_FIT, pflags)
        loc = [int(rng.next1() % 2) * 3 for _ in range(100)] if flags & E.FLAG_GANG_LOCALITY else None
        ga = a.preempt(allocs, prio, victims, gang_off=np.arange(0, 201, 2), locality=loc)
        gc = c.preempt(allocs, prio, victims, gang_off=np.arange(0, 201, 2), locality=loc)
        assert all(np.array_equal(x, y) for x, y in zip(ga, gc)), flags
        a.close()
        c.close()


def test_n1_refusals_and_states():
    """N1: isl_create's refusals and acceptances; N6: a few-node byte is EINVAL before the state, nothing changes; isl_place_gangs keeps
    its codes in every state (no profiles, no inventory, a snapshot, an empty partition; node scoring refuses open streams)."""
    lib = E.load_library()
    M, L = E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED
    for policy, flags, rc in ((E.POLICY_FIRST_FIT, SCORE, E.EINVAL), (E.POLICY_BEST_FIT, SCORE | E.FLAG_GANG_ONE_NODE, E.EINVAL),
                              (M, SCORE | E.FLAG_GANG_FEW_NODES, E.EINVAL), (L, SCORE | E.FLAG_GANG_MIN_MEMBERS, E.EINVAL),
                              (M, SCORE | E.FLAG_ALL_NODES, E.EINVAL), (M, SCORE | E.FLAG_GANG_ONE_NODE | E.FLAG_GANG_DISTINCT_NODES, E.EINVAL),
                              (M, SCORE | E.FLAG_GANG_LOCALITY | E.FLAG_GANG_ONE_NODE, E.EINVAL), (M, E.FLAG_GANG_ONE_NODE, E.EINVAL),
                              (L, E.FLAG_GANG_LOCALITY, E.EINVAL), (M, SCORE | E.FLAG_GANG_PREEMPT | E.FLAG_GANG_ONE_NODE, E.OK),
                              (L, SCORE | E.FLAG_GANG_DISTINCT_NODES, E.OK), (M, SCORE | E.FLAG_GANG_LOCALITY, E.OK), (L, SCORE, E.OK)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == rc, (policy, flags)
        if rc == E.OK:
            lib.isl_destroy(h)
    cfg = E.Config(E.ABI_VERSION, M, E.QUIRKS_REF_EXACT, -1, (1 << 20) + 1, 16, SCORE, 0)
    assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(ctypes.c_void_p())) == E.ERANGE
    rows = E.make_profiles(tables.A100_40GB)
    req = alloc_requests(np.zeros(4, dtype=np.uint8))
    out = np.zeros(4, dtype=E.RESULT_DTYPE)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)  # noqa: E731

    def call(eng, off, r=req):
        off = np.asarray(off, dtype=np.uint32)
        return lib.isl_place_gangs(eng._h, len(off) - 1, p(off), p(r), p(out))

    fresh = E.Engine(max_gpus=16, max_batch=16, policy=M, flags=SCORE | E.FLAG_GANG_LOCALITY)
    assert call(fresh, [0, 1]) == E.ESTATE
    fresh.load_profiles(rows)
    assert call(fresh, [0, 1]) == E.ESTATE
    few = req.copy()
    few["start"] = E.GANG_FEW_NODES
    assert call(fresh, [0, 2], few) == E.EINVAL                  # N6 comes before the state
    eng = engine(node_offsets(2, 2), rows, np.array([0x01, 0, 0, 0], dtype=np.uint8), M, SCORE | E.FLAG_GANG_LOCALITY, max_batch=3)
    assert call(eng, [0, 4]) == E.ERANGE
    assert call(eng, [0, 2, 2, 3]) == E.EINVAL
    eng.snapshot_occupancy()
    eng.reset_stats()
    before = (eng.read_occupancy().tolist(), eng.stats())
    assert call(eng, [0, 1, 3], few[:3]) == E.EINVAL
    with pytest.raises(ValueError):
        eng.place_gangs(req[:3], [0, 1, 3], [E.GANG_ONE_NODE, E.GANG_FEW_NODES])
    assert (eng.read_occupancy().tolist(), eng.stats()) == before
    assert eng.restore_occupancy() is None                       # the snapshot is still there
    assert call(eng, [0, 3], req[:3]) == E.OK and out["status"][:3].tolist() == [E.ST_PLACED] * 3
    eng.set_partition(1, 1)
    assert call(eng, [0, 1]) == E.ERANGE
    eng.close()
    eng = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), L, SCORE)
    with pytest.raises(E.EngineError):                           # node scoring opens no stream (rule 7), with the bit as without
        eng.stream_open(1)
    assert call(eng, [0, 2]) == E.OK
    eng.close()
    unflagged = engine(node_offsets(2, 2), rows, np.zeros(4, dtype=np.uint8), M, 0)
    assert call(unflagged, [0, 2]) == E.EINVAL                   # node scoring without the bit: unchanged
    unflagged.close()
    fresh.close()


def test_three_step_example():
    """The header's worked example: a MOST_ALLOCATED one-node engine puts [1g.10gb, 1g.10gb] on GPU 2 at starts 4 and 5."""
    rows = E.make_profiles(tables.H100_80GB)
    eng = engine(np.arange(4, dtype=np.uint32), rows, np.array([0x00, 0x3F, 0x0F], dtype=np.uint8), E.POLICY_MOST_ALLOCATED,
                 SCORE | E.FLAG_GANG_ONE_NODE)
    got = eng.place_gangs(alloc_requests(np.zeros(2, dtype=np.uint8)), [0, 2])
    assert [(int(r["gpu"]), int(r["start"])) for r in got] == [(2, 4), (2, 5)]
    eng.close()


@pytest.mark.parametrize("locality", LOCALITIES)
@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy, locality):
    """A 2^20-GPU partition of 8-GPU nodes (the cap), and 2^20 one-GPU nodes (node scoring's node cap)."""
    rng = SplitMix64(9600 + 10 * policy + locality)
    rows = E.make_profiles(tables.H100_80GB)
    for node_off in (np.arange(0, (1 << 20) + 1, 8, dtype=np.uint32), np.arange((1 << 20) + 1, dtype=np.uint32)):
        G = int(node_off[-1])
        occ = whole_bytes(rng, G, dense=True)
        req, off = random_call(rng, G, len(rows), 200, 6)
        if locality == GSO.PER_GANG:
            per = np.repeat(np.array([0, 1, 3])[(rng.next(len(off) - 1) % np.uint64(3)).astype(np.int64)], np.diff(off.astype(np.int64)))
            req["start"][req["op"] == E.OP_ALLOC] = per[req["op"] == E.OP_ALLOC]
        got = check((node_off, rows, None, occ, req, off, E.QUIRKS_REF_EXACT, policy, 0, G, locality), len(node_off))
        assert (got["status"] == E.ST_PLACED).any()


@pytest.mark.parametrize("case", LAYOUT_CASES)
def test_layout_edges(case):
    """Every edge of the CTA layout built from this device's SM count and k_ganglocal<per_gang, node_score>'s own shared-memory opt-in (its
    256 B of static shared memory), shares on both sides of the shared / global memory switch among them, 8 node tables of widths 4-8."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    assert edge(gang_plan(node_off, lo, hi, sms, optin - 256)), case
    i = LAYOUT_CASES.index(case)
    rows = t8tab()
    rng = SplitMix64(9700 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    off = small_gangs(rng, 400, 8)
    req = gang_call(rng, G, 16, 400)
    locs = np.array([0, 1, 3])[(rng.next(len(off) - 1) % np.uint64(3)).astype(np.int64)]
    per = np.repeat(locs, np.diff(off.astype(np.int64)))
    req["start"][req["op"] == E.OP_ALLOC] = per[req["op"] == E.OP_ALLOC]
    check((node_off, rows, node_table, whole_bytes(rng, G, dense=True), req, off, E.QUIRKS_FIXED, POLICIES[i % 2], lo, hi, GSO.PER_GANG),
          case)


@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
def test_table_limits(name, quirks):
    """16 profiles and 8 node tables: every fixture of the table-limit suite, every locality."""
    rows = FIXTURES[name]()
    rng = SplitMix64(9800 + CASES.index((name, quirks)))
    n_nodes = 300
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 8) for _ in range(n_nodes)]).astype(np.uint32)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes) if np.asarray(rows).ndim == 2 else None
    n_names = np.asarray(rows).shape[-1]
    for loc in LOCALITIES:
        req = gang_call(rng, G, n_names, 800)
        off = small_gangs(rng, 800, 6)
        if loc == GSO.PER_GANG:
            per = np.repeat(np.array([0, 1, 3])[(rng.next(len(off) - 1) % np.uint64(3)).astype(np.int64)], np.diff(off.astype(np.int64)))
            req["start"][req["op"] == E.OP_ALLOC] = per[req["op"] == E.OP_ALLOC]
        check((node_off, rows, node_table, whole_bytes(rng, G), req, off, quirks, POLICIES[loc % 2], 0, G, loc), (name, loc))


def test_place_pending_gangs_node_score():
    """A MostAllocated reconciler packs: a job joins the fuller node, replicas on distinct nodes take the fullest first; a
    LeastAllocated one spreads the job to the emptiest node."""
    for policy in POLICIES:
        items = cr_cluster([1, 1])
        r = ctl.InstasliceReconciler(items, policy=policy, gang_node_score=True, gang_locality=True)
        first = r.place_pending_gangs([pods(["1g.5gb"], "a")], locality=[E.GANG_ANY_NODES])
        assert first[0][0] == "placed"
        out = r.place_pending_gangs([pods(["1g.5gb", "1g.5gb"], "b"), pods(["2g.10gb", "2g.10gb"], "c")],
                                    locality=[E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES])
        assert [v for v, _ in out] == ["placed", "placed"]
        assert first[0][1][0]["nodename"] == "node-0"            # a tie between two empty nodes goes to the lower one
        assert {a["nodename"] for a in out[0][1]} == {"node-0" if policy == E.POLICY_MOST_ALLOCATED else "node-1"}
        assert len({a["nodename"] for a in out[1][1]}) == 2
        plain = ctl.InstasliceReconciler(cr_cluster([1, 1]), policy=policy, gang_node_score=True)
        assert plain.place_pending_gangs([pods(["1g.5gb", "1g.5gb"], "d")])[0][0] == "placed"


def test_host_mirror_gang_score_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_score_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_score_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
