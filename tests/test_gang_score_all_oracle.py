"""Every gang kind under node scoring (ISL_FLAG_GANG_NODE_SCORE | ISL_FLAG_GANG_NODE_SCORE_ALL, include/islplace.h C1-C8) on the CPU:
both checkers reproduce the known-answer vectors and agree with each other on random calls; the brute force has the consequences the
header states (C4 a-e, C5 through M5 a-b, C6 through B4 a-f) and equals the node-scored brute force of the parent engine where C7 says
nothing changes; the binding and isl_create accept and refuse what C1-C2 say."""
from __future__ import annotations

import ctypes
import types

import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests

import gang_balance_fast as GBF
import gang_locality_oracle as GLO
import gang_score_all_fast as GSA
import gang_score_all_oracle as GSAO
import gang_score_fast as GSF
import node_score_fast as NS
from test_gang_spread_oracle import random_cluster, random_gangs

POLICIES = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]
VECTORS = GSAO.kat_vectors()
ONE, FEW = E.GANG_ONE_NODE, E.GANG_FEW_NODES


def brute(node_off, rows, occ, req, off, policy, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0, hi=None, elastic=False,
          locality=GSA.PER_GANG):
    return GSA.place_gangs(node_off, rows, occ, req, off, policy, locality, quirks, node_table, lo, hi, elastic)


def with_bytes(req, off, locality):
    return GLO.with_locality(req, off, locality)


def random_bytes(rng, n_gangs, balanced_only=False):
    """One locality byte per gang: 0..3 or a balanced 4..7, and now and then a skew of 252."""
    b = (rng.next(n_gangs) % np.uint64(8)).astype(np.int64)
    if balanced_only:
        b |= 4
    b[rng.next(n_gangs) % np.uint64(11) == 0] = 255
    return b


def random_minima(rng, req, off):
    """A minimum byte 0..5 per gang in the ALLOC members' size."""
    req = req.copy()
    per = np.repeat((rng.next(len(off) - 1) % np.uint64(6)).astype(np.int64), np.diff(off.astype(np.int64)))
    req["size"][req["op"] == E.OP_ALLOC] = per[req["op"] == E.OP_ALLOC]
    return req


def same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def node_of(node_off, gpus):
    return np.searchsorted(node_off, np.asarray(gpus, dtype=np.int64), side="right") - 1


@pytest.mark.parametrize("checker", ["brute_force", "node_score_fast"])
@pytest.mark.parametrize("vector", VECTORS, ids=[v["name"] for v in VECTORS])
def test_kat(vector, checker):
    x = GSAO.vector_inputs(vector)
    want, occ_after, placed = GSAO.expected(vector)
    out, occ, n = GSAO.run_vector(GSA.place_gangs if checker == "brute_force" else GSAO.place_gangs, x)
    assert [tuple(int(v) for v in r) for r in out] == want
    assert occ.tolist() == occ_after.tolist()
    assert n == placed


def test_kat_holds_the_header_examples():
    """The worked examples of include/islplace.h C1-C8 are among the vectors, with the records the header states."""
    names = {v["name"] for v in VECTORS}
    for q in ("REF_EXACT", "FIXED"):
        for name in ("few MOST", "few LEAST", "one-node elastic m2 MOST", "one-node elastic m2 LEAST"):
            assert f"{name} {q}" in names
        for b in (4, 5):
            for pol in ("MOST_ALLOCATED", "LEAST_ALLOCATED"):
                assert f"balanced byte {b} {pol} {q}" in names


@pytest.mark.parametrize("elastic", [False, True])
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_checkers_agree(policy, quirks, n_tables, elastic):
    """Random calls: every locality byte, partitions that cut nodes, FREEs, NOOPs and unknown profiles, engine localities as well."""
    rng = SplitMix64(9100 + policy * 10 + quirks * 3 + n_tables + 100 * elastic)
    for trial in range(8):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 40, max_gang=8)
        loc = GSA.PER_GANG if trial % 4 else [E.GANG_ANY_NODES, ONE, FEW, E.GANG_DISTINCT_NODES][trial // 4 % 4 + (trial // 8) % 2]
        if loc is GSA.PER_GANG:
            req = with_bytes(req, off, random_bytes(rng, len(off) - 1))
        if elastic:
            req = random_minima(rng, req, off)
        a = brute(node_off, rows, occ, req, off, policy, quirks, node_table, lo, hi, elastic, loc)
        b = GSAO.place_gangs(node_off, rows, occ, req, off, policy, loc, quirks, node_table, lo, hi, elastic)
        bad = np.flatnonzero(a[0] != b[0])
        assert len(bad) == 0, (trial, bad[:4], a[0][bad[:4]], b[0][bad[:4]])
        assert np.array_equal(a[1], b[1]) and a[2] == b[2], trial


@pytest.mark.parametrize("policy", POLICIES)
def test_c7_bytes_0_1_3_equal_the_node_scored_engine(policy):
    """C7: without MIN, localities 0, 1 and 3 return what the engine without the bit returns (gang_score_fast)."""
    rng = SplitMix64(9200 + policy)
    for trial in range(12):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
        req, off = random_gangs(rng, int(node_off[-1]), n_names, 40, max_gang=6)
        req = with_bytes(req, off, [(0, 1, 3)[int(x)] for x in rng.next(len(off) - 1) % np.uint64(3)])
        a = brute(node_off, rows, occ, req, off, policy, E.QUIRKS_FIXED, node_table)
        b = GSF.place_gangs(node_off, rows, occ, req, off, policy, GSF.PER_GANG, E.QUIRKS_FIXED, node_table)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), trial


def one_gang(rng, n_names, max_members=8):
    return alloc_requests((rng.next(1 + int(rng.next1() % max_members)) % np.uint64(n_names)).astype(np.uint8))


@pytest.mark.parametrize("policy", POLICIES)
def test_c4ab_few_nodes_against_one_node(policy):
    """C4 (a): a few-node gang that some node takes whole gets the one-node gang's records and occupancy; (b) a few-node gang that
    fails fails as a one-node gang too."""
    rng = SplitMix64(9300 + policy)
    seen = [0, 0]
    for _ in range(40):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
        req = one_gang(rng, n_names)
        off = [0, len(req)]
        one = brute(node_off, rows, occ, with_bytes(req, off, [ONE]), off, policy, E.QUIRKS_FIXED, node_table)
        few = brute(node_off, rows, occ, with_bytes(req, off, [FEW]), off, policy, E.QUIRKS_FIXED, node_table)
        if one[2] == len(req):
            assert same(few, one)
            seen[0] += 1
        if few[2] < len(req):
            assert one[2] < len(req)
            seen[1] += 1
    assert min(seen) > 3, seen


@pytest.mark.parametrize("policy", POLICIES)
def test_c4c_c6c_one_node_is_first_fit(policy):
    """C4 (c) and C6 (c): on a one-node inventory, or a partition inside one node, few-node and balanced bytes equal a FIRST_FIT
    engine with the same gang flags; a balanced byte there equals byte 0 (B4 c)."""
    rng = SplitMix64(9400 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    for node_off, lo, hi in ((np.array([0, 24], np.uint32), 0, 24), (np.array([0, 5, 30, 33], np.uint32), 9, 27)):
        G = int(node_off[-1])
        occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
        for elastic in (False, True):
            req, off = random_gangs(rng, G, len(rows), 80, max_gang=8)
            req = with_bytes(req, off, np.where(rng.next(len(off) - 1) % np.uint64(2) == 0, FEW, random_bytes(rng, len(off) - 1, True)))
            if elastic:
                req = random_minima(rng, req, off)
            got = brute(node_off, rows, occ, req, off, policy, E.QUIRKS_REF_EXACT, None, lo, hi, elastic)
            want = GBF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, E.POLICY_FIRST_FIT, None, lo, hi, elastic=elastic)
            assert same(got, want)
            zero = brute(node_off, rows, occ, with_bytes(req, off, [0 if (b or 0) > 3 else (b or 0) for b in GLO.gang_localities(req, off)]), off,
                         policy, E.QUIRKS_REF_EXACT, None, lo, hi, elastic)
            assert same(got, zero)


@pytest.mark.parametrize("policy", POLICIES)
def test_c4d_c6d_gangs_of_one_equal_place_batch(policy):
    """C4 (d) and B4 (d): with gangs of one, few-node and balanced bytes equal isl_place_batch on the same engine (node_score_fast)."""
    rng = SplitMix64(9500 + policy)
    for _ in range(6):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
        req, _ = random_gangs(rng, int(node_off[-1]), n_names, 60)
        off = np.arange(len(req) + 1, dtype=np.uint32)
        got = brute(node_off, rows, occ, with_bytes(req, off, np.where(rng.next(len(req)) % np.uint64(2) == 0, FEW,
                                                                       random_bytes(rng, len(req), True))), off, policy, E.QUIRKS_FIXED,
                    node_table)
        want = NS.place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("policy", POLICIES)
def test_c4e_rounds_never_reuse_the_last_node(policy):
    """C4 (e): in a committed few-node gang the member after a maximal run on node N does not fit on N where the run left it."""
    rng = SplitMix64(9600 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    checked = 0
    for _ in range(400):
        node_off = np.cumsum([0] + [1 + int(rng.next1() % 2) for _ in range(1 + int(rng.next1() % 5))]).astype(np.uint32)
        G = int(node_off[-1])
        occ = (rng.next(G) & rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
        req = one_gang(rng, len(rows), 10)
        out, _, placed = brute(node_off, rows, occ, with_bytes(req, [0, len(req)], [FEW]), [0, len(req)], policy)
        if placed < len(req):
            continue
        nodes, cur = node_of(node_off, out["gpu"]), occ.copy()
        for j in range(len(req)):
            if j and nodes[j] != nodes[j - 1]:
                v = nodes[j - 1]
                alone = NS.place(node_off, rows, cur, req[j:j + 1], policy, lo=int(node_off[v]), hi=int(node_off[v + 1]))[0]
                assert alone["status"][0] != E.ST_PLACED
                checked += 1
            cur[out["gpu"][j]] |= ((1 << int(out["size"][j])) - 1) << int(out["start"][j])
    assert checked > 10


@pytest.mark.parametrize("policy", POLICIES)
def test_m5a_minimum_of_every_member_is_not_elastic(policy):
    """M5 (a) under C5: with every byte 0, or at least the gang's size, an elastic call equals the call without MIN."""
    rng = SplitMix64(9700 + policy)
    node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
    req, off = random_gangs(rng, int(node_off[-1]), n_names, 80, max_gang=8)
    req = with_bytes(req, off, random_bytes(rng, len(off) - 1))
    full = req.copy()
    full["size"][full["op"] == E.OP_ALLOC] = 0
    assert same(brute(node_off, rows, occ, full, off, policy, E.QUIRKS_FIXED, node_table, elastic=True),
                brute(node_off, rows, occ, req, off, policy, E.QUIRKS_FIXED, node_table))
    full["size"][full["op"] == E.OP_ALLOC] = 200
    assert same(brute(node_off, rows, occ, full, off, policy, E.QUIRKS_FIXED, node_table, elastic=True),
                brute(node_off, rows, occ, req, off, policy, E.QUIRKS_FIXED, node_table))


@pytest.mark.parametrize("policy", POLICIES)
def test_m5b_trimmed_gang_is_the_cut_gang(policy):
    """M5 (b) under C5: a gang trimmed at f gets the records and occupancy of its first f members placed without MIN, which commit."""
    rng = SplitMix64(9800 + policy)
    trims = 0
    for _ in range(150):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
        req = one_gang(rng, n_names)
        off = [0, len(req)]
        req = with_bytes(req, off, random_bytes(rng, 1))
        req["size"] = 1 + int(rng.next1() % 3)
        out, after, placed = brute(node_off, rows, occ, req, off, policy, E.QUIRKS_FIXED, node_table, elastic=True)
        if not 0 < placed < len(req):
            continue
        cut = req[:placed].copy()
        cut["size"] = 0
        want = brute(node_off, rows, occ, cut, [0, placed], policy, E.QUIRKS_FIXED, node_table)
        assert want[2] == placed and np.array_equal(out[:placed], want[0]) and np.array_equal(after, want[1])
        assert (out["status"][placed + 1:] == E.ST_GANG_TRIMMED).all()
        trims += 1
    assert trims > 10


@pytest.mark.parametrize("policy", POLICIES)
def test_c6_b4ab_balanced_against_distinct_and_any(policy):
    """B4 (a) under C6: a gang that commits whole with byte 3 (N4) gets the same records with byte 4; (b) byte 3 + k with k >= the
    gang's members equals byte 0 (N3)."""
    rng = SplitMix64(9900 + policy)
    seen = 0
    for _ in range(60):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
        req = one_gang(rng, n_names)
        off = [0, len(req)]
        d = brute(node_off, rows, occ, with_bytes(req, off, [3]), off, policy, E.QUIRKS_FIXED, node_table)
        if d[2] == len(req):
            assert same(brute(node_off, rows, occ, with_bytes(req, off, [4]), off, policy, E.QUIRKS_FIXED, node_table), d)
            seen += 1
        assert same(brute(node_off, rows, occ, with_bytes(req, off, [3 + len(req) + int(rng.next1() % 3)]), off, policy, E.QUIRKS_FIXED,
                          node_table),
                    brute(node_off, rows, occ, with_bytes(req, off, [0]), off, policy, E.QUIRKS_FIXED, node_table))
    assert seen > 5


@pytest.mark.parametrize("elastic", [False, True])
@pytest.mark.parametrize("policy", POLICIES)
def test_c6_b4e_gang_by_gang(policy, elastic):
    """B4 (e) under C6, and L3 (b): a call mixing every locality byte equals its gangs run one at a time."""
    rng = SplitMix64(10000 + policy + 10 * elastic)
    node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
    req, off = random_gangs(rng, int(node_off[-1]), n_names, 80, max_gang=8)
    req = with_bytes(req, off, random_bytes(rng, len(off) - 1))
    if elastic:
        req = random_minima(rng, req, off)
    got = brute(node_off, rows, occ, req, off, policy, E.QUIRKS_FIXED, node_table, elastic=elastic)
    alloc = req["op"] == E.OP_ALLOC
    frees = req.copy()
    frees["op"][alloc] = E.OP_NOOP
    out, cur, placed = brute(node_off, rows, occ, frees, [0, len(req)], policy, E.QUIRKS_FIXED, node_table)
    for a, b in zip(off[:-1], off[1:]):
        if not alloc[a:b].any():
            continue
        members = req[a:b].copy()
        members["op"][~alloc[a:b]] = E.OP_NOOP
        g, cur, n = brute(node_off, rows, cur, members, [0, b - a], policy, E.QUIRKS_FIXED, node_table, elastic=elastic)
        out[a:b][alloc[a:b]] = g[alloc[a:b]]
        placed += n
    assert same(got, (out, cur, placed))


@pytest.mark.parametrize("policy", POLICIES)
def test_c6_b4f_skew_1_evens_the_counts(policy):
    """B4 (f) under C6: k = 1 on nodes that admit every member to the end: the final per-node counts differ by at most 1."""
    rng = SplitMix64(10100 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    for n_nodes, members in ((6, 16), (5, 23), (7, 7)):
        node_off = np.cumsum([0] + [1 + int(rng.next1() % 3) for _ in range(n_nodes)]).astype(np.uint32)
        req = alloc_requests(np.zeros(members, dtype=np.uint8))
        got, _, placed = brute(node_off, rows, np.zeros(int(node_off[-1]), np.uint8), with_bytes(req, [0, members], [4]), [0, members],
                               policy)
        assert placed == members
        counts = np.bincount(node_of(node_off, got["gpu"]), minlength=n_nodes)
        assert counts.max() - counts.min() <= 1, counts


def _stub_engine(flags):
    eng = E.Engine.__new__(E.Engine)
    eng.flags = flags
    eng._h = None
    eng._lib = types.SimpleNamespace(isl_place_gangs=lambda *args: E.OK)
    return eng


def test_binding_accepts_few_node_bytes_with_the_bit():
    """C2: with FLAG_GANG_NODE_SCORE_ALL the binding passes a few-node locality on; without it the ValueError of N6 stays."""
    assert E.FLAG_GANG_NODE_SCORE_ALL == 16384
    S, L = E.FLAG_GANG_NODE_SCORE, E.FLAG_GANG_LOCALITY
    req = np.zeros(2, dtype=E.REQUEST_DTYPE)
    _stub_engine(S | L | E.FLAG_GANG_NODE_SCORE_ALL).place_gangs(req, [0, 1, 2], [ONE, FEW])
    _stub_engine(S | L | E.FLAG_GANG_BALANCED | E.FLAG_GANG_NODE_SCORE_ALL).place_gangs(req, [0, 1, 2], [FEW, 255])
    with pytest.raises(ValueError, match="few-node"):
        _stub_engine(S | L).place_gangs(req, [0, 1, 2], [ONE, FEW])


def _create(lib, policy, flags):
    cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
    h = ctypes.c_void_p()
    rc = lib.isl_create(ctypes.byref(cfg), ctypes.byref(h))
    if rc == E.OK:
        lib.isl_destroy(h)
    return rc


def test_create_codes_without_gpu():
    """C1: isl_create's argument checks for every combination of the gang flags, node scoring or not, with and without the bit: a
    refusal is ISL_EINVAL before any CUDA call; an accepted engine is OK, or ECUDA on a machine without a GPU."""
    lib = E.load_library()
    A, S = E.FLAG_GANG_NODE_SCORE_ALL, E.FLAG_GANG_NODE_SCORE
    one, dist, few, loc, mn, pre, bal = (E.FLAG_GANG_ONE_NODE, E.FLAG_GANG_DISTINCT_NODES, E.FLAG_GANG_FEW_NODES, E.FLAG_GANG_LOCALITY,
                                         E.FLAG_GANG_MIN_MEMBERS, E.FLAG_GANG_PREEMPT, E.FLAG_GANG_BALANCED)
    gang_flags = [one, dist, few, loc, mn, pre, bal, E.FLAG_ALL_NODES]
    for policy in (E.POLICY_FIRST_FIT, E.POLICY_MIN_FRAG, E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED):
        scoring = policy in (E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED)
        for mask in range(1 << len(gang_flags)):
            base = sum(f for i, f in enumerate(gang_flags) if mask >> i & 1)
            for flags in (base, base | S, base | S | A, base | A):
                localities = sum(bool(flags & f) for f in (one, dist, few, loc))
                ok = (localities <= 1
                      and not (flags & E.FLAG_ALL_NODES and (scoring or flags & (one | dist | few | loc | mn | pre | bal)))
                      and not (flags & A and not flags & S)
                      and not (flags & S and not scoring)
                      and not (scoring and flags & (one | dist | loc) and not flags & S)
                      and not (scoring and flags & (few | mn | bal) and not flags & A)
                      and not (flags & bal and not flags & loc)
                      and not (flags & pre and flags & (few | mn)))
                if ok and not flags & A:
                    continue                                 # accepted as before the bit; creating it would only cost time
                rc = _create(lib, policy, flags)
                assert (rc in (E.OK, E.ECUDA)) if ok else rc == E.EINVAL, (policy, flags, rc)
