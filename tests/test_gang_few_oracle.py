"""CPU checks of the few-node gang checkers (ISL_FLAG_GANG_FEW_NODES): the brute force (tests/gang_few_fast.cpp) and the restatements of
tests/gang_few_oracle.py reproduce the hand-worked vectors of tests/golden/kat_gang_few.json and agree with each other on random
clusters, and the brute force has the identities include/islplace.h states (F4 a-e) against the one-node brute force
(tests/gang_node_fast.cpp) and the unflagged gang rules (gang_oracle.fast_place_gangs)."""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests

import gang_few_fast as GFF
import gang_few_oracle as GFO
import gang_node_fast as GNF
import gang_oracle as GO
from range_oracle import RangeFast

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KAT = list(GFO.load_kat())


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


@pytest.mark.parametrize("place", [GFF.place_gangs, GFO.fast_gangs_few_nodes], ids=["brute_force", "range_fast"])
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
    for verdict, w in zip(GFO.ref_py_gangs_few_nodes(crs, pods, inputs["quirks"]), want):
        if w[0][3] == E.ST_PLACED:
            assert verdict[0] == "placed"
            assert [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in verdict[1]] == [r[:3] for r in w]
        else:
            assert verdict == ("aborted", next(k for k, r in enumerate(w) if r[3] != E.ST_GANG_ABORTED))
    assert GO.cr_occupancy(crs).tolist() == occ_after.tolist()


def random_cluster(rng, n_tables, max_nodes=12, max_gpus=6):
    """1..max_nodes nodes of 0..max_gpus GPUs (at least one GPU), dense occupancy, one or three per-node tables."""
    n_nodes = 1 + int(rng.next1() % max_nodes)
    sizes = [int(rng.next1() % (max_gpus + 1)) for _ in range(n_nodes)]
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


def random_gangs(rng, G, n_names, n, max_gang=8):
    """ALLOCs with a few unknown profiles, FREEs and NOOPs mixed into gangs of 1..max_gang requests."""
    req = alloc_requests((rng.next(n) % np.uint64(n_names)).astype(np.uint8))
    req["profile"][rng.next(n) % np.uint64(41) == 0] = E.PROFILE_UNKNOWN
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
    split = 0
    for trial in range(6):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 80)
        a, occ_a, rounds = GFF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi, rounds=True)
        b, occ_b = GFO.fast_gangs_few_nodes(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
        bad = np.flatnonzero(a != b)
        assert len(bad) == 0, (trial, bad[:4], a[bad[:4]], b[bad[:4]])
        assert np.array_equal(occ_a, occ_b), trial
        split += int((rounds > 0).sum())
    assert split > 0                                # some gang needed more than one round


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_ref_py_agrees_first_fit(quirks):
    rng = SplitMix64(950 + quirks)
    names = [r[0] for r in tables.A100_40GB]
    rows = E.make_profiles(tables.A100_40GB)
    for trial in range(5):
        node_off, _rows, occ, _t, _n = random_cluster(rng, 1)
        gangs = [[int(rng.next1() % len(names)) for _ in range(1 + int(rng.next1() % 6))] for _ in range(8)]
        crs = GO.cluster_crs(node_off, np.zeros(len(node_off) - 1, np.uint8), occ, [tables.A100_40GB])
        pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, names[p]) for k, p in enumerate(g)]
                for i, g in enumerate(gangs)]
        verdicts = GFO.ref_py_gangs_few_nodes(crs, pods, quirks)
        cur = occ
        for g, (verdict, detail) in zip(gangs, verdicts):
            out, cur = GFF.place_gangs(node_off, rows, cur, alloc_requests(np.asarray(g, dtype=np.uint8)), [0, len(g)], quirks)
            if verdict == "placed":
                assert [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in detail] == \
                    [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in out], trial
                assert (out["status"] == E.ST_PLACED).all()
            else:
                assert int(np.flatnonzero(out["status"] != E.ST_GANG_ABORTED)[0]) == detail, trial
        assert np.array_equal(GO.cr_occupancy(crs), cur), trial


@pytest.mark.parametrize("policy", POLICIES)
def test_one_node_gangs_agree_gang_by_gang(policy):
    """F4 (a) and (b), gang by gang from the same state: a gang a GANG_ONE_NODE engine commits gets the same records and occupancy here,
    and a gang that aborts here aborts there."""
    rng = SplitMix64(60 + policy)
    seen = {"one": 0, "split": 0, "abort": 0}
    for trial in range(4):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 1 + 2 * (trial % 2), max_nodes=8, max_gpus=4)
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 80, 10)
        for a, b in zip(off[:-1], off[1:]):
            one, occ_one = GNF.place_gangs(node_off, rows, occ, req[a:b], [0, b - a], E.QUIRKS_REF_EXACT, policy, node_table)
            few, occ_few = GFF.place_gangs(node_off, rows, occ, req[a:b], [0, b - a], E.QUIRKS_REF_EXACT, policy, node_table)
            alloc = req["op"][a:b] == E.OP_ALLOC
            if alloc.any() and (one["status"][alloc] == E.ST_PLACED).all():
                assert np.array_equal(few, one) and np.array_equal(occ_few, occ_one), (trial, a)
                seen["one"] += 1
            elif alloc.any() and (few["status"][alloc] == E.ST_PLACED).all():
                seen["split"] += 1
            elif alloc.any():
                assert not (one["status"][alloc] == E.ST_PLACED).all()
                assert np.array_equal(occ_few, occ_one), (trial, a)       # both: the frees only
                seen["abort"] += 1
            occ = occ_few
    assert min(seen.values()) > 0, seen


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_one_node_equals_unflagged(policy, quirks):
    """F4 (c): on an inventory of one node, and on a partition inside one node, the unflagged gang rules' records and occupancy."""
    rng = SplitMix64(31 + policy * 2 + quirks)
    rows = E.make_profiles(tables.H100_80GB)
    for G, node_off, part in ((1, [0, 1], None), (5, [0, 5], None), (64, [0, 64], None), (40, [0, 10, 30, 40], (12, 27))):
        node_off = np.asarray(node_off, dtype=np.uint32)
        lo, hi = part or (0, G)
        occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
        req, off = random_gangs(rng, G, len(rows), 60)
        got, occ_got = GFF.place_gangs(node_off, rows, occ, req, off, quirks, policy, None, lo, hi)
        ref = RangeFast(node_off, rows, occ, lo, hi, quirks, policy)
        want = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows))
        assert np.array_equal(got, want), G
        assert np.array_equal(occ_got, ref.occupancy()), G


@pytest.mark.parametrize("policy", POLICIES)
def test_gangs_of_one(policy):
    """F4 (d): with gangs of one, a GANG_ONE_NODE call; under first-fit and right-to-left also isl_place_batch."""
    rng = SplitMix64(77 + policy)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(20)]).astype(np.uint32)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.H100_80GB)
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_gangs(rng, G, len(rows), 200)
    off = np.arange(len(req) + 1)
    got, occ_got = GFF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
    one, occ_one = GNF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
    assert np.array_equal(got, one) and np.array_equal(occ_got, occ_one)
    if policy in (E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT):
        ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
        ref.load(occ)
        assert np.array_equal(got, ref.place(req))
        assert np.array_equal(occ_got, ref.occupancy())


def same_node_runs(node_of, got, idx):
    """The maximal runs of consecutive ALLOC members (request indices idx) on one node, as lists of positions in idx."""
    runs = []
    for k, i in enumerate(idx):
        n = node_of(int(got["gpu"][i]))
        if runs and runs[-1][0] == n:
            runs[-1][1].append(k)
        else:
            runs.append((n, [k]))
    return [r for _n, r in runs]


@pytest.mark.parametrize("policy", POLICIES)
def test_rounds_are_the_same_node_runs(policy):
    """F4 (e): the maximal same-node runs of a committed gang's ALLOC members are exactly its rounds."""
    rng = SplitMix64(90 + policy)
    multi = 0
    for trial in range(4):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 1 + 2 * (trial % 2), max_nodes=10, max_gpus=3)
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 120, 12)
        got, _occ, rounds = GFF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy, node_table, rounds=True)
        node_of = lambda g: int(np.searchsorted(node_off, g, side="right")) - 1  # noqa: E731
        for a, b in zip(off[:-1], off[1:]):
            idx = [i for i in range(a, b) if req["op"][i] == E.OP_ALLOC]
            if not idx or got["status"][idx[0]] != E.ST_PLACED:
                continue
            by_round = {}
            for k, i in enumerate(idx):
                by_round.setdefault(int(rounds[i]), []).append(k)
            assert same_node_runs(node_of, got, idx) == [by_round[r] for r in sorted(by_round)], (trial, a)
            multi += len(by_round) > 1
    assert multi > 0
