"""CPU checks of the one-node gang checkers (ISL_FLAG_GANG_ONE_NODE): the brute force (tests/gang_node_fast.cpp) and the restatements of
tests/gang_node_oracle.py reproduce the hand-worked vectors of tests/golden/kat_gang_node.json and agree with each other on random
clusters, and the brute force has the identities include/islplace.h states (G4)."""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests

import gang_node_fast as GNF
import gang_node_oracle as GNO
import gang_oracle as GO

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KAT = list(GNO.load_kat())


def run_kat(place, inputs, gangs):
    """One call per gang, as the vectors are worked; returns the records per gang and the final occupancy."""
    occ = inputs["occ"]
    lo, hi = inputs["partition"] or (0, int(inputs["node_off"][-1]))
    got = []
    for gang in gangs:
        req = alloc_requests(np.asarray(gang, dtype=np.uint8))
        out, occ = place(inputs["node_off"], inputs["rows"], occ, req, [0, len(req)], inputs["quirks"], inputs["policy"],
                         inputs["node_table"], lo, hi)
        got.append([tuple(int(x) for x in r) for r in out])
    return got, occ


@pytest.mark.parametrize("place", [GNF.place_gangs, GNO.fast_gangs_one_node], ids=["brute_force", "range_fast"])
@pytest.mark.parametrize("kat", KAT, ids=[k[0] for k in KAT])
def test_kat(place, kat):
    _name, inputs, gangs, want, occ_after = kat
    got, occ = run_kat(place, inputs, gangs)
    assert got == want
    assert occ.tolist() == occ_after.tolist()


@pytest.mark.parametrize("kat", [k for k in KAT if k[1]["policy"] == E.POLICY_FIRST_FIT and k[1]["partition"] is None],
                         ids=lambda k: k[0])
def test_kat_ref_py(kat):
    """First-fit vectors on custom-resource dicts, member by member with the reference's own search on one node's resource."""
    _name, inputs, gangs, want, occ_after = kat
    table_list = [getattr(tables, t) for t in inputs["table_names"]]
    names = [r[0] for r in table_list[0]] if len(table_list) == 1 else list(E.make_profile_tables(table_list)[0])
    node_table = inputs["node_table"] if inputs["node_table"] is not None else np.zeros(len(inputs["node_off"]) - 1, np.uint8)
    crs = GO.cluster_crs(inputs["node_off"], node_table, inputs["occ"], table_list)
    pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, names[p] if p < len(names) else "no-such-profile")
             for k, p in enumerate(g)] for i, g in enumerate(gangs)]
    for verdict, w in zip(GNO.ref_py_gangs_one_node(crs, pods, inputs["quirks"]), want):
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


def random_gangs(rng, G, n_names, n):
    req = alloc_requests((rng.next(n) % np.uint64(n_names + 1)).astype(np.uint8))
    req["profile"][req["profile"] == n_names] = E.PROFILE_UNKNOWN
    for i in np.flatnonzero(rng.next(n) % np.uint64(9) == 0):
        start = int(rng.next1() % 8)
        req[i] = (int(rng.next1() % (G + 2)), 0, E.OP_FREE, start, 1 + int(rng.next1() % (8 - start)))
    req["op"][rng.next(n) % np.uint64(23) == 0] = E.OP_NOOP
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % 5)))
    return req, np.asarray(off, dtype=np.uint32)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_checkers_agree(policy, quirks, n_tables):
    rng = SplitMix64(500 + policy * 10 + quirks * 3 + n_tables)
    for trial in range(6):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 40)
        a, occ_a = GNF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
        b, occ_b = GNO.fast_gangs_one_node(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
        bad = np.flatnonzero(a != b)
        assert len(bad) == 0, (trial, bad[:4], a[bad[:4]], b[bad[:4]])
        assert np.array_equal(occ_a, occ_b), trial


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_ref_py_agrees_first_fit(quirks):
    rng = SplitMix64(900 + quirks)
    names = [r[0] for r in tables.A100_40GB]
    for trial in range(5):
        node_off, _rows, occ, _t, _n = random_cluster(rng, 1)
        rows = E.make_profiles(tables.A100_40GB)
        gangs = [[int(rng.next1() % len(names)) for _ in range(1 + int(rng.next1() % 4))] for _ in range(8)]
        crs = GO.cluster_crs(node_off, np.zeros(len(node_off) - 1, np.uint8), occ, [tables.A100_40GB])
        pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, names[p]) for k, p in enumerate(g)]
                for i, g in enumerate(gangs)]
        verdicts = GNO.ref_py_gangs_one_node(crs, pods, quirks)
        cur = occ
        for g, (verdict, detail) in zip(gangs, verdicts):
            out, cur = GNF.place_gangs(node_off, rows, cur, alloc_requests(np.asarray(g, dtype=np.uint8)), [0, len(g)], quirks)
            if verdict == "placed":
                assert [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in detail] == \
                    [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in out], trial
                assert (out["status"] == E.ST_PLACED).all()
            else:
                assert int(np.flatnonzero(out["status"] != E.ST_GANG_ABORTED)[0]) == detail, trial
        assert np.array_equal(GO.cr_occupancy(crs), cur), trial


@pytest.mark.parametrize("policy", POLICIES)
def test_one_node_equals_unflagged(policy):
    """G4: on an inventory of one node the brute force gives the unflagged gang rules' records and occupancy."""
    rng = SplitMix64(31 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    for G in (1, 5, 64):
        node_off = np.array([0, G], dtype=np.uint32)
        occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
        req, off = random_gangs(rng, G, len(rows), 60)
        got, occ_got = GNF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
        ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
        ref.load(occ)
        want = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows))
        assert np.array_equal(got, want), G
        assert np.array_equal(occ_got, ref.occupancy()), G


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_gangs_of_one_equal_place_batch(policy):
    """G4: with gangs of one, first-fit and right-to-left one-node gangs are isl_place_batch."""
    rng = SplitMix64(77 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(20)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_gangs(rng, G, len(rows), 200)
    got, occ_got = GNF.place_gangs(node_off, rows, occ, req, np.arange(len(req) + 1), E.QUIRKS_REF_EXACT, policy)
    ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
    ref.load(occ)
    assert np.array_equal(got, ref.place(req))
    assert np.array_equal(occ_got, ref.occupancy())
