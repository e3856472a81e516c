"""CPU checks of the elastic-gang checkers (ISL_FLAG_GANG_MIN_MEMBERS): the direct brute force tests/gang_min_fast.cpp and the
compositions by truncation of tests/gang_min_oracle.py reproduce the hand-worked vectors of tests/golden/kat_gang_min.json and agree on
random clusters; the brute force has the identities include/islplace.h states (M5 a, b, d); and the argument checks of M1 / M6 that need
no engine."""
import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import gang_locality_oracle as GLO
import gang_min_fast as GMF
import gang_min_oracle as GMO
import gang_oracle as GO
from instaslice_b200.workloads import SplitMix64, alloc_requests
from test_gang_few_oracle import random_cluster, random_gangs

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KAT = list(GMO.load_kat())


def random_minima(rng, off, most=6):
    """0..most per gang: 0 and values at or above a gang's size mean every member, the rest trim or abort."""
    return (rng.next(len(off) - 1) % np.uint64(most + 1)).astype(np.int64)


@pytest.mark.parametrize("kat", KAT, ids=[k[0] for k in KAT])
def test_kat_both_checkers(kat):
    _name, inp, req, off, want, occ_after, placed = kat
    lo, hi = inp["partition"] or (0, int(inp["node_off"][-1]))
    args = (inp["node_off"], inp["rows"], inp["occ"], req, off, inp["locality"], inp["quirks"], inp["policy"], inp["node_table"], lo, hi)
    for got, occ, n in (GMF.place_gangs(*args), GMO.fast_gangs_min(*args)):
        assert [tuple(int(x) for x in r) for r in got] == want
        assert occ.tolist() == occ_after.tolist()
        assert n == placed


def ref_py_call(inp, occ, gangs, locality, minima):
    table_list = [getattr(tables, t) for t in inp["table_names"]]
    node_table = inp["node_table"] if inp["node_table"] is not None else np.zeros(len(inp["node_off"]) - 1, np.uint8)
    crs = GO.cluster_crs(inp["node_off"], node_table, occ, table_list)
    pods = [[({"uid": "p%d-%d" % (i, k), "name": "p", "namespace": "default"}, name) for k, name in enumerate(g)] for i, g in enumerate(gangs)]
    return GMO.ref_py_gangs_min(crs, pods, locality, minima, inp["quirks"]), GO.cr_occupancy(crs)


def check_verdicts(verdicts, got, off):
    """The ref_py verdicts against the engine-shaped records of one call."""
    for verdict, a, b in zip(verdicts, off[:-1], off[1:]):
        rec = got[a:b]
        placed = [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in rec if r["status"] == E.ST_PLACED]
        if verdict[0] == "aborted":
            assert not placed and int(np.flatnonzero(rec["status"] != E.ST_GANG_ABORTED)[0]) == verdict[1]
            continue
        assert [(int(x["gpuUUID"][4:]), x["start"], x["size"]) for x in verdict[1]] == placed
        if verdict[0] == "trimmed":
            f = verdict[2]
            assert len(placed) == f and rec["status"][f] in (E.ST_NO_CAPACITY, E.ST_BAD_PROFILE)
            assert (rec["status"][f + 1:] == E.ST_GANG_TRIMMED).all()
        else:
            assert len(placed) == len(rec)


@pytest.mark.parametrize("kat", [k for k in KAT if k[1]["policy"] == E.POLICY_FIRST_FIT and k[1]["partition"] is None and
                                 all(isinstance(m, str) and m in k[1]["names"] for g in k[1]["gangs"] for m in g)], ids=lambda k: k[0])
def test_kat_ref_py(kat):
    """First-fit vectors with known profiles and no FREEs or NOOPs on custom-resource dicts."""
    _name, inp, _req, off, want, occ_after, _placed = kat
    verdicts, occ = ref_py_call(inp, inp["occ"], inp["gangs"], inp["locality"], inp["min_members"])
    got = np.array([(g, s, z, st) for g, s, z, st in want], dtype=E.RESULT_DTYPE)
    check_verdicts(verdicts, got, off)
    assert occ.tolist() == occ_after.tolist()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_brute_force_equals_truncation(policy, quirks, n_tables):
    """The direct brute force and composition (i) on random clusters, localities and minima, FREEs, NOOPs, unknown profiles and cut
    partitions included: records, occupancy and members placed."""
    rng = SplitMix64(2100 + policy * 10 + quirks * 3 + n_tables)
    seen = set()
    for trial in range(6):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables)
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else sorted(int(x) for x in (rng.next1() % (G + 1), rng.next1() % (G + 1)))
        if lo == hi:
            lo, hi = 0, G
        req, off = random_gangs(rng, G, n_names, 80)
        locality = (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64)
        req = GMO.with_minimum(req, off, random_minima(rng, off))
        a, occ_a, n_a = GMF.place_gangs(node_off, rows, occ, req, off, locality, quirks, policy, node_table, lo, hi)
        b, occ_b, n_b = GMO.fast_gangs_min(node_off, rows, occ, req, off, locality, quirks, policy, node_table, lo, hi)
        bad = np.flatnonzero(a != b)
        assert len(bad) == 0, (trial, bad[:4], a[bad[:4]], b[bad[:4]])
        assert np.array_equal(occ_a, occ_b) and n_a == n_b, trial
        seen |= set(np.unique(a["status"]).tolist())
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_GANG_TRIMMED, E.ST_NO_CAPACITY} <= seen


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_compositions_agree_first_fit(quirks, n_tables):
    """The brute force and composition (ii) (ref_py on custom-resource dicts) on random clusters, localities and minima, first-fit,
    ALLOCs of known profiles only."""
    rng = SplitMix64(2200 + quirks * 7 + n_tables)
    trimmed = 0
    for trial in range(5):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, n_tables, max_nodes=8, max_gpus=4)
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 40, 6)
        req["op"] = E.OP_ALLOC
        req["profile"][req["profile"] == E.PROFILE_UNKNOWN] = 0
        locality = (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64)
        minima = random_minima(rng, off)
        got, occ_i, _ = GMF.place_gangs(node_off, rows, occ, GMO.with_minimum(req, off, minima), off, locality, quirks, E.POLICY_FIRST_FIT,
                                        node_table)
        if n_tables == 1:
            names = [r[0] for r in tables.H100_80GB]
            inp = {"table_names": ["H100_80GB"], "node_table": None, "node_off": node_off, "quirks": quirks}
        else:
            names = list(E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])[0])
            inp = {"table_names": ["A100_40GB", "H100_80GB", "A30_24GB"], "node_table": node_table, "node_off": node_off, "quirks": quirks}
        gangs = [[names[int(p)] for p in req["profile"][a:b]] for a, b in zip(off[:-1], off[1:])]
        verdicts, occ_ii = ref_py_call(inp, occ, gangs, locality, minima.tolist())
        check_verdicts(verdicts, got, off)
        assert occ_ii.tolist() == occ_i.tolist(), trial
        trimmed += sum(v[0] == "trimmed" for v in verdicts)
    assert trimmed > 0


def unflagged(node_off, rows, occ, req, off, loc, quirks, policy, node_table, lo, hi):
    """The call on the checker of locality ``loc`` without the flag: the locality composition, whose checkers never read the size byte."""
    plain = req.copy()
    plain["size"][plain["op"] == E.OP_ALLOC] = 0
    return GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(plain, off, [loc] * (len(off) - 1)), off, quirks, policy,
                                   node_table, lo, hi)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("loc", GLO.LOCALITIES)
def test_m5a_zero_or_large_minima_equal_unflagged(policy, loc):
    """M5 (a): every byte 0, or every byte at least its gang's k, gives the call without the flag."""
    rng = SplitMix64(2300 + policy * 5 + loc)
    for trial in range(3):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 1 + 2 * (trial % 2))
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 80)
        want, occ_want = unflagged(node_off, rows, occ, req, off, loc, E.QUIRKS_REF_EXACT, policy, node_table, 0, G)
        k = np.add.reduceat(req["op"] == E.OP_ALLOC, off[:-1].astype(np.int64)).astype(np.int64)
        for minima in (np.zeros(len(off) - 1, np.int64), k + (rng.next(len(k)) % np.uint64(3)).astype(np.int64)):
            got, occ_got, n = GMF.place_gangs(node_off, rows, occ, GMO.with_minimum(req, off, minima), off, loc, E.QUIRKS_REF_EXACT, policy,
                                              node_table)
            assert np.array_equal(got, want) and np.array_equal(occ_got, occ_want), trial
            assert n == int(((want["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)).sum())


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("loc", GLO.LOCALITIES)
def test_m5b_trimmed_gang_equals_cut_gang(policy, loc):
    """M5 (b): every gang the brute force trims at f gets exactly the records and occupancy of the gang cut to its first f ALLOC members
    without the flag, and that cut gang commits."""
    rng = SplitMix64(2400 + policy * 5 + loc)
    trimmed = 0
    for trial in range(4):
        node_off, rows, occ, node_table, n_names = random_cluster(rng, 1 + 2 * (trial % 2))
        G = int(node_off[-1])
        req, off = random_gangs(rng, G, n_names, 60, 10)
        req["op"][req["op"] == E.OP_FREE] = E.OP_NOOP
        cur = occ.copy()
        for a, b in zip(off[:-1], off[1:]):
            gang = req[a:b].copy()
            k = int((gang["op"] == E.OP_ALLOC).sum())
            gang = GMO.with_minimum(gang, [0, b - a], [1 + int(rng.next1() % max(k, 1))])
            got, after, _ = GMF.place_gangs(node_off, rows, cur, gang, [0, b - a], loc, E.QUIRKS_REF_EXACT, policy, node_table)
            idx = np.flatnonzero(gang["op"] == E.OP_ALLOC)
            f = int((got["status"][idx] == E.ST_PLACED).sum())
            if 0 < f < k:                                   # trimmed: some ALLOC members placed, not all
                assert (got["status"][idx[:f]] == E.ST_PLACED).all(), trial
                cut, cut_after = unflagged(node_off, rows, cur, gang[idx[:f]], [0, f], loc, E.QUIRKS_REF_EXACT, policy, node_table, 0, G)
                assert (cut["status"] == E.ST_PLACED).all() and np.array_equal(cut, got[idx[:f]]), trial
                assert np.array_equal(cut_after, after), trial
                trimmed += 1
            cur = after
    assert trimmed > 0


@pytest.mark.parametrize("policy", POLICIES)
def test_m5d_gangs_of_one(policy):
    """M5 (d): gangs of one ALLOC member are unaffected by any byte."""
    rng = SplitMix64(2500 + policy)
    node_off, rows, occ, node_table, n_names = random_cluster(rng, 3, max_nodes=20)
    G = int(node_off[-1])
    req, off = random_gangs(rng, G, n_names, 200, 1)
    for loc in GLO.LOCALITIES:
        want, occ_want = unflagged(node_off, rows, occ, req, off, loc, E.QUIRKS_REF_EXACT, policy, node_table, 0, G)
        minima = (rng.next(len(off) - 1) % np.uint64(256)).astype(np.int64)
        got, occ_got, _ = GMF.place_gangs(node_off, rows, occ, GMO.with_minimum(req, off, minima), off, loc, E.QUIRKS_REF_EXACT, policy,
                                          node_table)
        assert np.array_equal(got, want) and np.array_equal(occ_got, occ_want), loc


def test_m1_effective_minimum_and_m6_mixed_bytes():
    """M1: m' = k for m = 0 or m >= k, else m; a FREE's size is its span and a NOOP's is ignored.  M6: two ALLOC members of one gang with
    different bytes are refused."""
    req = np.zeros(7, dtype=E.REQUEST_DTYPE)
    req["op"] = [E.OP_ALLOC, E.OP_FREE, E.OP_ALLOC, E.OP_NOOP, E.OP_ALLOC, E.OP_ALLOC, E.OP_ALLOC]
    req["size"] = [2, 5, 2, 9, 255, 255, 0]
    assert GMF.effective_minimum(req, [0, 4, 6, 7]).tolist() == [2, 2, 1]
    req["size"][2] = 3
    with pytest.raises(ValueError):
        GMF.effective_minimum(req, [0, 4, 6, 7])
    assert GMF.effective_minimum(req[1:2], [0, 1]).tolist() == [0]      # no ALLOC member: no minimum


def test_m7_leading_run_not_best_subset():
    """M7 on three GPUs, two with slice 0 busy: [4g.20gb x3, 1g.5gb x2] stops at the second 4g.20gb, so with m = 1 only the first member
    commits and with m = 2 the gang aborts, although the first 4g.20gb and both 1g.5gb would fit."""
    rows = E.make_profiles(tables.A100_40GB)
    node_off = np.array([0, 1, 2, 3], dtype=np.uint32)
    occ = np.array([0x01, 0x01, 0x00], dtype=np.uint8)
    profiles = np.array([3, 3, 3, 0, 0], dtype=np.uint8)                                   # 4g.20gb x3, 1g.5gb x2
    got, occ_got, n = GMF.place_gangs(node_off, rows, occ, GMO.with_minimum(alloc_requests(profiles), [0, 5], [1]), [0, 5], E.GANG_ANY_NODES)
    assert got["status"].tolist() == [E.ST_PLACED, E.ST_NO_CAPACITY, E.ST_GANG_TRIMMED, E.ST_GANG_TRIMMED, E.ST_GANG_TRIMMED]
    assert n == 1 and occ_got.tolist() == [0x01, 0x01, 0x0F]
    got, occ_got, n = GMF.place_gangs(node_off, rows, occ, GMO.with_minimum(alloc_requests(profiles), [0, 5], [2]), [0, 5], E.GANG_ANY_NODES)
    assert n == 0 and (got["status"] != E.ST_PLACED).all() and occ_got.tolist() == occ.tolist()
