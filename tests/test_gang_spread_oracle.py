"""CPU checks of the distinct-node gang checkers (ISL_FLAG_GANG_DISTINCT_NODES): the brute force (tests/gang_spread_fast.cpp) and the
restatements of tests/gang_spread_oracle.py reproduce the hand-worked vectors of tests/golden/kat_gang_spread.json and agree with each
other on random clusters, and the brute force has the consequences include/islplace.h states (S5)."""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests

import gang_oracle as GO
import gang_spread_fast as GSF
import gang_spread_oracle as GSO

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KAT = list(GSO.load_kat())


def run_kat(place, inputs, gangs):
    """One call per gang, as the vectors are worked; returns the records per gang and the final occupancy."""
    occ = inputs["occ"]
    lo, hi = inputs["partition"] or (0, int(inputs["node_off"][-1]))
    got = []
    for req in gangs:
        out, occ = place(inputs["node_off"], inputs["rows"], occ, req, [0, len(req)], inputs["quirks"], inputs["policy"],
                         inputs["node_table"], lo, hi)
        got.append([tuple(int(x) for x in r) for r in out])
    return got, occ


@pytest.mark.parametrize("place", [GSF.place_gangs, GSO.fast_gangs_distinct_nodes], ids=["brute_force", "range_fast"])
@pytest.mark.parametrize("kat", KAT, ids=[k[0] for k in KAT])
def test_kat(place, kat):
    _name, inputs, gangs, want, occ_after, _plain = kat
    got, occ = run_kat(place, inputs, gangs)
    assert got == want
    assert occ.tolist() == occ_after.tolist()


@pytest.mark.parametrize("kat", [k for k in KAT if k[1]["policy"] == E.POLICY_FIRST_FIT and k[1]["partition"] is None
                                 and all(g is not None for g in k[5])], ids=lambda k: k[0])
def test_kat_ref_py(kat):
    """First-fit vectors of profile names only, on custom-resource dicts with the reference's own node loop per member."""
    _name, inputs, _gangs, want, occ_after, plain = kat
    table_list = [getattr(tables, t) for t in inputs["table_names"]]
    node_table = inputs["node_table"] if inputs["node_table"] is not None else np.zeros(len(inputs["node_off"]) - 1, np.uint8)
    crs = GO.cluster_crs(inputs["node_off"], node_table, inputs["occ"], table_list)
    pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, name) for k, name in enumerate(g)]
            for i, g in enumerate(plain)]
    for verdict, w in zip(GSO.ref_py_gangs_distinct_nodes(crs, pods, inputs["quirks"]), want):
        if w[0][3] == E.ST_PLACED:
            assert verdict[0] == "placed"
            assert [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in verdict[1]] == [r[:3] for r in w]
        else:
            assert verdict == ("aborted", next(k for k, r in enumerate(w) if r[3] != E.ST_GANG_ABORTED))
    assert GO.cr_occupancy(crs).tolist() == occ_after.tolist()


def random_cluster(rng, n_tables):
    """1..12 nodes of 0..6 GPUs (at least one GPU), dense occupancy, one or three per-node tables."""
    n_nodes = 1 + int(rng.next1() % 12)
    sizes = [int(rng.next1() % 7) for _ in range(n_nodes)]
    sizes[int(rng.next1() % n_nodes)] += 1
    node_off = np.cumsum([0] + sizes).astype(np.uint32)
    G = int(node_off[-1])
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    if n_tables == 1:
        rows, node_table = E.make_profiles(tables.H100_80GB), None
        n_names = len(rows)
    else:
        names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
        node_table = (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8)
        n_names = len(names)
    return node_off, rows, occ, node_table, n_names


def random_gangs(rng, G, n_names, n, max_gang=5):
    req = alloc_requests((rng.next(n) % np.uint64(n_names + 1)).astype(np.uint8))
    req["profile"][req["profile"] == n_names] = E.PROFILE_UNKNOWN
    for i in np.flatnonzero(rng.next(n) % np.uint64(9) == 0):
        start = int(rng.next1() % 8)
        req[i] = (int(rng.next1() % (G + 2)), 0, E.OP_FREE, start, 1 + int(rng.next1() % (8 - start)))
    req["op"][rng.next(n) % np.uint64(23) == 0] = E.OP_NOOP
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % max_gang)))
    return req, np.asarray(off, dtype=np.uint32)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_checkers_agree(policy, quirks, n_tables):
    rng = SplitMix64(700 + policy * 10 + quirks * 3 + n_tables)
    for trial in range(6):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 40)
        a, occ_a = GSF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
        b, occ_b = GSO.fast_gangs_distinct_nodes(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
        bad = np.flatnonzero(a != b)
        assert len(bad) == 0, (trial, bad[:4], a[bad[:4]], b[bad[:4]])
        assert np.array_equal(occ_a, occ_b), trial


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_ref_py_agrees_first_fit(quirks):
    rng = SplitMix64(950 + quirks)
    names = [r[0] for r in tables.A100_40GB]
    rows = E.make_profiles(tables.A100_40GB)
    for trial in range(5):
        node_off, _rows, occ, _t, _n = random_cluster(rng, 1)
        gangs = [[int(rng.next1() % len(names)) for _ in range(1 + int(rng.next1() % 4))] for _ in range(8)]
        crs = GO.cluster_crs(node_off, np.zeros(len(node_off) - 1, np.uint8), occ, [tables.A100_40GB])
        pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, names[p]) for k, p in enumerate(g)]
                for i, g in enumerate(gangs)]
        verdicts = GSO.ref_py_gangs_distinct_nodes(crs, pods, quirks)
        cur = occ
        for g, (verdict, detail) in zip(gangs, verdicts):
            out, cur = GSF.place_gangs(node_off, rows, cur, alloc_requests(np.asarray(g, dtype=np.uint8)), [0, len(g)], quirks)
            if verdict == "placed":
                assert [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in detail] == \
                    [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in out], trial
                assert (out["status"] == E.ST_PLACED).all()
            else:
                assert int(np.flatnonzero(out["status"] != E.ST_GANG_ABORTED)[0]) == detail, trial
        assert np.array_equal(GO.cr_occupancy(crs), cur), trial


@pytest.mark.parametrize("policy", POLICIES)
def test_gangs_of_one_equal_place_batch(policy):
    """S5 (a): with gangs of one the brute force is isl_place_batch, on every policy."""
    rng = SplitMix64(77 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(20)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_gangs(rng, G, len(rows), 200)
    got, occ_got = GSF.place_gangs(node_off, rows, occ, req, np.arange(len(req) + 1), E.QUIRKS_REF_EXACT, policy)
    ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
    ref.load(occ)
    assert np.array_equal(got, ref.place(req))
    assert np.array_equal(occ_got, ref.occupancy())


@pytest.mark.parametrize("policy", POLICIES)
def test_one_node_inventory_aborts_gangs_of_two(policy):
    """S5 (c): on one node every gang of two or more ALLOC members aborts; when member 0 places, member 1 reports NO_CAPACITY."""
    rng = SplitMix64(131 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.array([0, 64], dtype=np.uint32)
    occ = (rng.next(64) & np.uint64(0x3F)).astype(np.uint8)
    req, off = random_gangs(rng, 64, len(rows), 200, max_gang=6)
    got, _ = GSF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
    seen = 0
    for a, b in zip(off[:-1], off[1:]):
        idx = np.flatnonzero(req["op"][a:b] == E.OP_ALLOC) + a
        if len(idx) >= 2:
            assert (got["status"][idx] != E.ST_PLACED).all()
            if int(req["profile"][idx[0]]) < len(rows) and got["status"][idx[0]] == E.ST_GANG_ABORTED:
                known = int(req["profile"][idx[1]]) < len(rows)
                assert got["status"][idx[1]] == (E.ST_NO_CAPACITY if known else E.ST_BAD_PROFILE)
                seen += known
    assert seen > 0


@pytest.mark.parametrize("policy", POLICIES)
def test_whole_gpu_profiles_on_one_gpu_nodes_equal_unflagged(policy):
    """S5 (d): one-GPU nodes, ISL_QUIRKS_FIXED, every profile of size 8: the brute force equals the unflagged gang rules."""
    rng = SplitMix64(171 + policy)
    rows = E.make_profiles([("7g.80gb", 8, [0], 4), ("7g.80gb-b", 8, [0], 5)])
    G = 300
    node_off = np.arange(G + 1, dtype=np.uint32)
    occ = np.where(rng.next(G) % np.uint64(3) == 0, 0, (rng.next(G) & np.uint64(0xFF))).astype(np.uint8)
    req, off = random_gangs(rng, G, len(rows), 400, max_gang=8)
    got, occ_got = GSF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_FIXED, policy)
    ref = oracle.Fast(node_off, rows, E.QUIRKS_FIXED, policy)
    ref.load(occ)
    want = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows))
    assert np.array_equal(got, want)
    assert np.array_equal(occ_got, ref.occupancy())
    assert (got["status"] == E.ST_PLACED).any() and (got["status"] == E.ST_GANG_ABORTED).any()
