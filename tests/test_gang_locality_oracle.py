"""CPU checks of the per-gang locality checkers (ISL_FLAG_GANG_LOCALITY): composition (i) of tests/gang_locality_oracle.py (the brute
forces of each locality) and composition (ii) (the ref_py restatements on custom-resource dicts) agree on random clusters, both reproduce
the hand-worked vectors of tests/golden/kat_gang_locality.json, and composition (i) has the identities include/islplace.h states (L3 a-c)
against the brute force of each locality alone and oracle.Fast."""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64

import gang_few_fast as GFF
import gang_locality_oracle as GLO
import gang_node_fast as GNF
import gang_oracle as GO
import gang_spread_fast as GSF
from range_oracle import RangeFast
from test_gang_few_oracle import random_cluster, random_gangs

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KAT = list(GLO.load_kat())


def alone(loc, node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi):
    """The call on the checker of one locality, as an engine created with that locality's flag (none for 0) answers it."""
    if loc == E.GANG_ANY_NODES:
        table = np.zeros(len(node_off) - 1, np.uint8) if node_table is None else node_table
        ref = RangeFast(node_off, rows, occ, lo, hi, quirks, policy, node_table=table if np.asarray(rows).ndim == 2 else None)
        return GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows, table)), ref.occupancy()
    brute = {E.GANG_ONE_NODE: GNF, E.GANG_FEW_NODES: GFF, E.GANG_DISTINCT_NODES: GSF}[loc]
    return brute.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)


@pytest.mark.parametrize("kat", KAT, ids=[k[0] for k in KAT])
def test_kat_composition(kat):
    _name, inp, req, off, want, occ_after = kat
    lo, hi = inp["partition"] or (0, int(inp["node_off"][-1]))
    got, occ = GLO.fast_gangs_locality(inp["node_off"], inp["rows"], inp["occ"], req, off, inp["quirks"], inp["policy"], inp["node_table"],
                                       lo, hi)
    assert [tuple(int(x) for x in r) for r in got] == want
    assert occ.tolist() == occ_after.tolist()


def ref_py_call(inp, occ, gangs, locality):
    """Composition (ii) on the vector's cluster: (verdicts, occupancy after)."""
    table_list = [getattr(tables, t) for t in inp["table_names"]]
    node_table = inp["node_table"] if inp["node_table"] is not None else np.zeros(len(inp["node_off"]) - 1, np.uint8)
    crs = GO.cluster_crs(inp["node_off"], node_table, occ, table_list)
    pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, name) for k, name in enumerate(g)] for i, g in enumerate(gangs)]
    return GLO.ref_py_gangs_locality(crs, pods, locality, inp["quirks"]), GO.cr_occupancy(crs)


@pytest.mark.parametrize("kat", [k for k in KAT if k[1]["policy"] == E.POLICY_FIRST_FIT and k[1]["partition"] is None and
                                 all(isinstance(m, str) for g in k[1]["gangs"] for m in g)], ids=lambda k: k[0])
def test_kat_ref_py(kat):
    """First-fit vectors without FREEs on custom-resource dicts, each gang on the ref_py restatement of its locality."""
    _name, inp, _req, off, want, occ_after = kat
    verdicts, occ = ref_py_call(inp, inp["occ"], inp["gangs"], inp["locality"])
    for verdict, a, b in zip(verdicts, off[:-1], off[1:]):
        w = want[a:b]
        if w[0][3] == E.ST_PLACED:
            assert verdict[0] == "placed"
            assert [(int(x["gpuUUID"][4:]), x["start"], x["size"]) for x in verdict[1]] == [r[:3] for r in w]
        else:
            assert verdict == ("aborted", next(k for k, r in enumerate(w) if r[3] != E.ST_GANG_ABORTED))
    assert occ.tolist() == occ_after.tolist()


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_compositions_agree_first_fit(quirks, n_tables):
    """(i) and (ii) on random clusters, random localities, first-fit, no FREEs (the ref_py restatements take ALLOCs only)."""
    rng = SplitMix64(1200 + quirks * 7 + n_tables)
    for trial in range(5):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables, max_nodes=8, max_gpus=4)
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 40, 5)
        req["op"] = E.OP_ALLOC
        req["profile"][req["profile"] == E.PROFILE_UNKNOWN] = 0
        locality = (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64)
        got, occ_i = GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(req, off, locality), off, quirks, E.POLICY_FIRST_FIT,
                                             node_table)
        if n_tables == 1:
            names = [r[0] for r in tables.H100_80GB]
            inp = {"table_names": ["H100_80GB"], "node_table": None, "node_off": node_off, "quirks": quirks}
        else:
            names = list(E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])[0])
            inp = {"table_names": ["A100_40GB", "H100_80GB", "A30_24GB"], "node_table": node_table, "node_off": node_off, "quirks": quirks}
        gangs = [[names[int(p)] for p in req["profile"][a:b]] for a, b in zip(off[:-1], off[1:])]
        verdicts, occ_ii = ref_py_call(inp, occ, gangs, locality)
        for verdict, a, b in zip(verdicts, off[:-1], off[1:]):
            rec = got[a:b]
            if (rec["status"] == E.ST_PLACED).all():
                assert verdict[0] == "placed", (trial, a)
                assert [(int(x["gpuUUID"][4:]), x["start"], x["size"]) for x in verdict[1]] == \
                    [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in rec], (trial, a)
            else:
                assert verdict == ("aborted", int(np.flatnonzero(rec["status"] != E.ST_GANG_ABORTED)[0])), (trial, a)
        assert occ_ii.tolist() == occ_i.tolist(), trial


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_l3a_each_locality_alone(policy, quirks, n_tables):
    """L3 (a): a call whose gangs all carry locality k equals the checker of k alone, FREEs, NOOPs, unknown profiles and partitions
    included."""
    rng = SplitMix64(1300 + policy * 10 + quirks * 3 + n_tables)
    for trial in range(3):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 60)
        for loc in GLO.LOCALITIES:
            a, occ_a = GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(req, off, [loc] * (len(off) - 1)), off, quirks, policy,
                                               node_table, lo, hi)
            b, occ_b = alone(loc, node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
            assert np.array_equal(a, b) and np.array_equal(occ_a, occ_b), (trial, loc)


@pytest.mark.parametrize("policy", POLICIES)
def test_l3b_gang_by_gang(policy):
    """L3 (b): a call equals its gangs one at a time on the checker of each one's locality, after the call's FREEs, with the occupancy
    handed on."""
    rng = SplitMix64(1400 + policy)
    for trial in range(4):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 1 + 2 * (trial % 2))
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 60)
        locality = (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64)
        got, occ_got = GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(req, off, locality), off, E.QUIRKS_REF_EXACT, policy,
                                               node_table)
        frees = req.copy()
        frees["op"][frees["op"] == E.OP_ALLOC] = E.OP_NOOP
        want, cur = alone(0, node_off, rows, occ, frees, [0, len(req)], E.QUIRKS_REF_EXACT, policy, node_table, 0, G)
        for g, (a, b) in enumerate(zip(off[:-1], off[1:])):
            idx = np.flatnonzero(req["op"][a:b] == E.OP_ALLOC) + a
            if len(idx):
                want[idx], cur = alone(int(locality[g]), node_off, rows, cur, req[idx], [0, len(idx)], E.QUIRKS_REF_EXACT, policy, node_table,
                                       0, G)
        assert np.array_equal(got, want) and np.array_equal(occ_got, cur), trial


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_l3c_any_node_gangs_of_one(policy):
    """L3 (c): with every byte 0, gangs of one equal isl_place_batch (oracle.Fast)."""
    rng = SplitMix64(1500 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = np.cumsum([0] + [1 + int(rng.next1() % 6) for _ in range(40)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    req, _ = random_gangs(rng, G, len(rows), 400, 1)
    got, occ_got = GLO.fast_gangs_locality(node_off, rows, occ, req, np.arange(len(req) + 1), E.QUIRKS_REF_EXACT, policy)
    ref = RangeFast(node_off, rows, occ, 0, G, E.QUIRKS_REF_EXACT, policy)
    assert np.array_equal(got, ref.place(req)) and np.array_equal(occ_got, ref.occupancy())
    if policy == E.POLICY_FIRST_FIT:
        fast = oracle.Fast(node_off, rows)
        fast.load(occ)
        assert np.array_equal(got, fast.place(req))


def test_l6_one_node_gang_of_one_under_best_fit():
    """L6: under best-fit a one-node gang of one takes the best GPU of the first node that admits it, a locality-0 gang the best GPU."""
    rows = E.make_profiles(tables.A100_40GB)
    node_off, occ = np.array([0, 1, 3], dtype=np.uint32), np.array([0x00, 0x00, 0xFC], dtype=np.uint8)
    req = np.zeros(1, dtype=E.REQUEST_DTYPE)
    for loc, gpu in ((E.GANG_ONE_NODE, 0), (E.GANG_FEW_NODES, 0), (E.GANG_ANY_NODES, 2), (E.GANG_DISTINCT_NODES, 2)):
        got, _ = GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(req, [0, 1], [loc]), [0, 1], E.QUIRKS_REF_EXACT,
                                         E.POLICY_BEST_FIT)
        assert int(got["gpu"][0]) == gpu, loc
