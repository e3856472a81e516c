"""CPU checks of the balanced-gang checkers (ISL_FLAG_GANG_BALANCED): the brute force (tests/gang_balance_fast.cpp) and the
restatements of tests/gang_balance_oracle.py reproduce the hand-worked vectors of tests/golden/kat_gang_balance.json and agree with each
other on random clusters; the brute force has the consequences include/islplace.h states (B4); the binding and isl_create refuse what
B1 and B6 refuse."""
import copy
import ctypes

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests

import gang_balance_fast as GBF
import gang_balance_oracle as GBO
import gang_locality_oracle as GLO
import gang_oracle as GO
from test_gang_spread_oracle import random_cluster, random_gangs

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KAT = list(GBO.load_kat())


def brute(node_off, rows, occ, req, off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None, lo=0, hi=None,
          elastic=False):
    return GBF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, elastic=elastic)


def with_bytes(req, off, locality):
    return GLO.with_locality(req, off, locality)


@pytest.mark.parametrize("checker", ["brute_force", "range_fast"])
@pytest.mark.parametrize("kat", KAT, ids=[k[0] for k in KAT])
def test_kat(kat, checker):
    _name, inputs, req, off, want, occ_after, placed = kat
    lo, hi = inputs["partition"] or (0, int(inputs["node_off"][-1]))
    place = GBF.place_gangs if checker == "brute_force" else GBO.fast_gangs_balance
    got, occ, n = place(inputs["node_off"], inputs["rows"], inputs["occ"], req, off, inputs["quirks"], inputs["policy"],
                        inputs["node_table"], lo, hi, elastic=inputs["elastic"])
    assert [tuple(int(x) for x in r) for r in got] == want
    assert occ.tolist() == occ_after.tolist()
    assert n == placed


@pytest.mark.parametrize("kat", [k for k in KAT if k[1]["policy"] == E.POLICY_FIRST_FIT and k[1]["partition"] is None
                                 and not k[1]["elastic"] and min(k[1]["locality"]) > E.GANG_DISTINCT_NODES], ids=lambda k: k[0])
def test_kat_ref_py(kat):
    """First-fit balanced vectors on custom-resource dicts with the reference's own node loop per member."""
    _name, inputs, _req, off, want, occ_after, _placed = kat
    table_list = [getattr(tables, t) for t in inputs["table_names"]]
    node_table = inputs["node_table"] if inputs["node_table"] is not None else np.zeros(len(inputs["node_off"]) - 1, np.uint8)
    crs = GO.cluster_crs(inputs["node_off"], node_table, inputs["occ"], table_list)
    pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, name) for k, name in enumerate(g)]
            for i, g in enumerate(inputs["gangs"])]
    verdicts = GBO.ref_py_gangs_balance(crs, pods, [b - E.GANG_DISTINCT_NODES for b in inputs["locality"]], inputs["quirks"])
    for verdict, a, b in zip(verdicts, off[:-1], off[1:]):
        w = want[a:b]
        if w[0][3] == E.ST_PLACED:
            assert verdict[0] == "placed"
            assert [(int(x["gpuUUID"][4:]), x["start"], x["size"]) for x in verdict[1]] == [r[:3] for r in w]
        else:
            assert verdict == ("aborted", next(k for k, r in enumerate(w) if r[3] != E.ST_GANG_ABORTED))
    assert GO.cr_occupancy(crs).tolist() == occ_after.tolist()


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


@pytest.mark.parametrize("elastic", [False, True])
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_checkers_agree(policy, quirks, n_tables, elastic):
    rng = SplitMix64(4100 + policy * 10 + quirks * 3 + n_tables + 100 * elastic)
    for trial in range(6):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 40, max_gang=8)
        req = with_bytes(req, off, random_bytes(rng, len(off) - 1))
        if elastic:
            req = random_minima(rng, req, off)
        a, occ_a, pa = brute(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, elastic)
        b, occ_b, pb = GBO.fast_gangs_balance(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, elastic)
        bad = np.flatnonzero(a != b)
        assert len(bad) == 0, (trial, bad[:4], a[bad[:4]], b[bad[:4]])
        assert np.array_equal(occ_a, occ_b), trial
        assert pa == pb, trial


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_ref_py_agrees_first_fit(quirks):
    rng = SplitMix64(4300 + quirks)
    names = [r[0] for r in tables.A100_40GB]
    rows = E.make_profiles(tables.A100_40GB)
    for trial in range(5):
        node_off, _rows, occ, _t, _n = random_cluster(rng, 1)
        gangs = [[int(rng.next1() % len(names)) for _ in range(1 + int(rng.next1() % 6))] for _ in range(8)]
        skews = [1 + int(rng.next1() % 3) for _ in gangs]
        crs = GO.cluster_crs(node_off, np.zeros(len(node_off) - 1, np.uint8), occ, [tables.A100_40GB])
        pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, names[p]) for k, p in enumerate(g)]
                for i, g in enumerate(gangs)]
        verdicts = GBO.ref_py_gangs_balance(crs, pods, skews, quirks)
        cur = occ
        for g, k, (verdict, detail) in zip(gangs, skews, verdicts):
            req = alloc_requests(np.asarray(g, dtype=np.uint8))
            out, cur, _ = brute(node_off, rows, cur, with_bytes(req, [0, len(g)], [E.gang_balanced_nodes(k)]), [0, len(g)], quirks)
            if verdict == "placed":
                assert [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in detail] == \
                    [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in out], trial
                assert (out["status"] == E.ST_PLACED).all()
            else:
                assert int(np.flatnonzero(out["status"] != E.ST_GANG_ABORTED)[0]) == detail, trial
        assert np.array_equal(GO.cr_occupancy(crs), cur), trial


def gang_by_gang(node_off, rows, occ, req, off, quirks, policy, node_table=None, lo=0, hi=None, elastic=False):
    """B4 (e): the call's FREEs, then each gang alone with the occupancy handed on."""
    alloc = req["op"] == E.OP_ALLOC
    frees = req.copy()
    frees["op"][alloc] = E.OP_NOOP
    out, cur, placed = brute(node_off, rows, occ, frees, [0, len(req)], quirks, policy, node_table, lo, hi)
    for a, b in zip(off[:-1], off[1:]):
        if not alloc[a:b].any():
            continue
        members = req[a:b].copy()
        members["op"][~alloc[a:b]] = E.OP_NOOP
        got, cur, n = brute(node_off, rows, cur, members, [0, b - a], quirks, policy, node_table, lo, hi, elastic)
        out[a:b][alloc[a:b]] = got[alloc[a:b]]
        placed += n
    return out, cur, placed


@pytest.mark.parametrize("policy", POLICIES)
def test_b4a_committed_distinct_gangs_equal_byte_4(policy):
    """B4 (a): a gang that commits whole with byte 3 gets the same records with byte 4."""
    rng = SplitMix64(4400 + policy)
    node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 4) for _ in range(30)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
    node_table = (rng.next(30) % np.uint64(3)).astype(np.uint8)
    seen = 0
    for _ in range(60):
        req = alloc_requests((rng.next(1 + int(rng.next1() % 6)) % np.uint64(n_names)).astype(np.uint8))
        off = [0, len(req)]
        d, occ_d, _ = brute(node_off, rows, occ, with_bytes(req, off, [3]), off, E.QUIRKS_FIXED, policy, node_table)
        if (d["status"] == E.ST_PLACED).all():
            b, occ_b, _ = brute(node_off, rows, occ, with_bytes(req, off, [4]), off, E.QUIRKS_FIXED, policy, node_table)
            assert np.array_equal(b, d) and np.array_equal(occ_b, occ_d)
            occ, seen = occ_d, seen + 1
    assert seen > 10


@pytest.mark.parametrize("policy", POLICIES)
def test_b4b_skew_at_least_the_gang_is_byte_0(policy):
    """B4 (b): byte 3 + k with k >= the gang's ALLOC count equals byte 0, over a whole call."""
    rng = SplitMix64(4500 + policy)
    node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
    req, off = random_gangs(rng, int(node_off[-1]), n_names, 60, max_gang=8)
    k = np.add.reduceat((req["op"] == E.OP_ALLOC).astype(np.int64), off[:-1].astype(np.int64))
    skew = np.maximum(k, 1) + (rng.next(len(k)) % np.uint64(3)).astype(np.int64)
    a = brute(node_off, rows, occ, with_bytes(req, off, 3 + skew), off, E.QUIRKS_FIXED, policy, node_table)
    b = brute(node_off, rows, occ, with_bytes(req, off, np.zeros(len(k), np.int64)), off, E.QUIRKS_FIXED, policy, node_table)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


@pytest.mark.parametrize("policy", POLICIES)
def test_b4c_one_node_is_byte_0(policy):
    """B4 (c): on a one-node inventory, and on a partition inside one node, every balanced byte equals byte 0."""
    rng = SplitMix64(4600 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    for node_off, lo, hi in ((np.array([0, 24], np.uint32), 0, 24), (np.array([0, 5, 30, 33], np.uint32), 9, 27)):
        G = int(node_off[-1])
        occ = (rng.next(G) & rng.next(G) & np.uint64(0x7F)).astype(np.uint8)
        req, off = random_gangs(rng, G, len(rows), 80, max_gang=8)
        want = brute(node_off, rows, occ, with_bytes(req, off, np.zeros(len(off) - 1, np.int64)), off, E.QUIRKS_REF_EXACT, policy,
                     None, lo, hi)
        got = brute(node_off, rows, occ, with_bytes(req, off, random_bytes(rng, len(off) - 1, True)), off, E.QUIRKS_REF_EXACT, policy,
                    None, lo, hi)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]


@pytest.mark.parametrize("policy", POLICIES)
def test_b4d_gangs_of_one(policy):
    """B4 (d): gangs of one equal byte 0, and under FIRST_FIT and RIGHT_TO_LEFT isl_place_batch."""
    rng = SplitMix64(4700 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(20)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_gangs(rng, G, len(rows), 200)
    off = np.arange(len(req) + 1, dtype=np.uint32)
    got = brute(node_off, rows, occ, with_bytes(req, off, random_bytes(rng, len(req), True)), off, E.QUIRKS_REF_EXACT, policy)
    zero = brute(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
    assert np.array_equal(got[0], zero[0]) and np.array_equal(got[1], zero[1])
    if policy in (E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT):
        ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
        ref.load(occ)
        assert np.array_equal(got[0], ref.place(req))
        assert np.array_equal(got[1], ref.occupancy())


@pytest.mark.parametrize("elastic", [False, True])
@pytest.mark.parametrize("policy", POLICIES)
def test_b4e_gang_by_gang(policy, elastic):
    """B4 (e): a call mixing every locality equals its gangs run one at a time."""
    rng = SplitMix64(4800 + policy + 10 * elastic)
    node_off, rows, occ, node_table, n_names = random_cluster(rng, 3)
    G = int(node_off[-1])
    req, off = random_gangs(rng, G, n_names, 80, max_gang=8)
    req = with_bytes(req, off, random_bytes(rng, len(off) - 1))
    if elastic:
        req = random_minima(rng, req, off)
    got = brute(node_off, rows, occ, req, off, E.QUIRKS_FIXED, policy, node_table, elastic=elastic)
    want = gang_by_gang(node_off, rows, occ, req, off, E.QUIRKS_FIXED, policy, node_table, elastic=elastic)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]) and got[2] == want[2]


@pytest.mark.parametrize("policy", POLICIES)
def test_b4f_skew_1_evens_the_counts(policy):
    """B4 (f): k = 1 on nodes that admit every member to the end: the final per-node counts differ by at most 1."""
    rng = SplitMix64(4900 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    for n_nodes, members in ((6, 16), (5, 23), (7, 7)):
        sizes = [1 + int(rng.next1() % 3) for _ in range(n_nodes)]
        node_off = np.cumsum([0] + sizes).astype(np.uint32)
        req = alloc_requests(np.zeros(members, dtype=np.uint8))
        got, _, placed = brute(node_off, rows, np.zeros(int(node_off[-1]), np.uint8), with_bytes(req, [0, members], [4]), [0, members],
                               E.QUIRKS_REF_EXACT, policy)
        assert placed == members
        counts = np.bincount(np.searchsorted(node_off, got["gpu"].astype(np.int64), side="right") - 1, minlength=n_nodes)
        assert counts.max() - counts.min() <= 1, counts


def test_balanced_nodes_binding():
    """B1: gang_balanced_nodes maps maxSkew 1..252 to bytes 4..255 and refuses the rest."""
    assert E.gang_balanced_nodes(1) == 4 and E.gang_balanced_nodes(252) == 255
    for bad in (0, 253, -1, 1.5, True):
        with pytest.raises(ValueError):
            E.gang_balanced_nodes(bad)
    assert E.FLAG_GANG_BALANCED == 8192


def test_create_refusals_without_gpu():
    """B6: isl_create refuses the flag without per-gang locality, under node scoring or with ISL_FLAG_ALL_NODES, before any CUDA call."""
    lib = E.load_library()
    B, L = E.FLAG_GANG_BALANCED, E.FLAG_GANG_LOCALITY
    for policy, flags in ((E.POLICY_FIRST_FIT, B), (E.POLICY_BEST_FIT, B | E.FLAG_GANG_DISTINCT_NODES),
                          (E.POLICY_MOST_ALLOCATED, B | L), (E.POLICY_LEAST_ALLOCATED, B | L | E.FLAG_GANG_NODE_SCORE),
                          (E.POLICY_FIRST_FIT, B | L | E.FLAG_ALL_NODES), (E.POLICY_FIRST_FIT, B | L | E.FLAG_GANG_ONE_NODE)):
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        assert lib.isl_create(ctypes.byref(cfg), ctypes.byref(h)) == E.EINVAL, (policy, flags)
    for flags in (B | L, B | L | E.FLAG_GANG_MIN_MEMBERS, B | L | E.FLAG_GANG_PREEMPT):
        cfg = E.Config(E.ABI_VERSION, E.POLICY_MIN_FRAG, E.QUIRKS_REF_EXACT, -1, 16, 16, flags, 0)
        h = ctypes.c_void_p()
        rc = lib.isl_create(ctypes.byref(cfg), ctypes.byref(h))
        assert rc in (E.OK, E.ECUDA), flags                  # accepted: without a GPU it fails at its first CUDA call
        if rc == E.OK:
            lib.isl_destroy(h)
