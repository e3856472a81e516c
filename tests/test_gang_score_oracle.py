"""Node-scored gangs (ISL_FLAG_GANG_NODE_SCORE, include/islplace.h N1-N8) on the CPU: the hand-worked vectors of
tests/golden/kat_gang_score.json on both checkers, the two checkers (tests/gang_score_fast.cpp and the composition over node_score_fast in
tests/gang_score_oracle.py) agreeing on random clusters, N8 (a)-(d) on the checkers, and N6's locality-byte refusal in the binding."""
import random

import numpy as np
import pytest

from instaslice_b200 import engine as E

import gang_node_fast as GNF
import gang_score_fast as GSF
import gang_score_oracle as GSO
import gang_spread_fast as GSPF
import node_score_fast as NS

CHECKERS = {"fast": GSF.place_gangs, "oracle": GSO.place_gangs}
POLICIES = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]


@pytest.mark.parametrize("checker", list(CHECKERS))
@pytest.mark.parametrize("case", GSO.kat_cases(), ids=lambda c: c["name"])
def test_kat(case, checker):
    inp = GSO.case_inputs(case)
    want, occ_after = GSO.expected(case)
    out, occ, placed = GSO.run(CHECKERS[checker], inp)
    assert [tuple(int(x) for x in r) for r in out] == [tuple(w) for w in want], case["why"]
    assert occ.tolist() == occ_after.tolist()
    assert placed == sum(1 for r in want if r[3] == E.ST_PLACED)


@pytest.mark.parametrize("locality", [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GSO.PER_GANG])
@pytest.mark.parametrize("policy", POLICIES)
def test_checkers_agree(policy, locality):
    """Random clusters: one to three node tables, both quirk sets, partitions that cut nodes, FREEs, NOOPs and unknown profiles."""
    rnd = random.Random(7100 + 10 * policy + locality)
    for _ in range(150):
        _, rows = GSO.random_rows(rnd)
        inp = GSO.random_case(rnd, rnd.randint(1, 24), rnd.randint(1, 16), rows, locality=locality, policy=policy)
        a, b = GSO.run(GSF.place_gangs, inp), GSO.run(GSO.place_gangs, inp)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def _inputs(rnd, locality, policy, gangs_of_one=False):
    _, rows = GSO.random_rows(rnd)
    node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, loc = GSO.random_case(rnd, rnd.randint(1, 24), rnd.randint(1, 16), rows,
                                                                                           max_gang=1 if gangs_of_one else 4,
                                                                                           locality=locality, policy=policy)
    return node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, loc


@pytest.mark.parametrize("policy", POLICIES)
def test_n8a_gangs_of_one_equal_place_batch(policy):
    """N8 (a): with gangs of one ALLOC member, every locality equals node scoring's isl_place_batch: records, occupancy, placed."""
    rnd = random.Random(7200 + policy)
    for loc in (E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GSO.PER_GANG):
        for _ in range(60):
            node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, loc = _inputs(rnd, loc, policy, gangs_of_one=True)
            out, occ_g, placed = GSF.place_gangs(node_off, rows, occ, req, off, policy, loc, quirks, node_table, lo, hi)
            want, occ_b = NS.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
            assert np.array_equal(out, want) and np.array_equal(occ_g, occ_b)
            assert placed == int((want["status"] == E.ST_PLACED).sum())


@pytest.mark.parametrize("policy", POLICIES)
def test_n8b_any_node_gang_by_gang(policy):
    """N8 (b): under any-node locality a committed gang equals node scoring's isl_place_batch of its ALLOC members on the occupancy
    before it, and an aborted gang changes nothing."""
    rnd = random.Random(7300 + policy)
    for _ in range(100):
        node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, loc = _inputs(rnd, E.GANG_ANY_NODES, policy)
        out, occ_after, _ = GSF.place_gangs(node_off, rows, occ, req, off, policy, loc, quirks, node_table, lo, hi)
        _, cur = NS.place(node_off, rows, occ, req[req["op"] != E.OP_ALLOC], policy, quirks, node_table, lo, hi)
        for a, b in zip(off[:-1], off[1:]):
            alloc = np.flatnonzero(req["op"][a:b] == E.OP_ALLOC) + a
            if len(alloc) == 0:
                continue
            want, nxt = NS.place(node_off, rows, cur, req[alloc], policy, quirks, node_table, lo, hi)
            if (out["status"][alloc] == E.ST_PLACED).all():
                assert np.array_equal(out[alloc], want)
                cur = nxt
            else:
                assert not (out["status"][alloc] == E.ST_PLACED).any()
        assert np.array_equal(occ_after, cur)


@pytest.mark.parametrize("policy", POLICIES)
def test_n8c_one_node_is_first_fit(policy):
    """N8 (c): on a one-node inventory, or a partition inside one node, a flagged call equals isl_place_gangs on a FIRST_FIT engine with
    the same locality: the one-node and distinct-node brute forces of those engines (any node on one node is a one-node gang, G4)."""
    rnd = random.Random(7400 + policy)
    for loc in (E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES):
        for _ in range(60):
            node_off, rows, node_table, occ, req, off, quirks, policy, _lo, _hi, _ = _inputs(rnd, loc, policy)
            v = rnd.randrange(len(node_off) - 1)
            lo, hi = int(node_off[v]), int(node_off[v + 1])
            if lo == hi:
                continue
            lo2 = rnd.randint(lo, hi - 1)
            hi2 = rnd.randint(lo2 + 1, hi)
            out, occ_g, _ = GSF.place_gangs(node_off, rows, occ, req, off, policy, loc, quirks, node_table, lo2, hi2)
            if loc == E.GANG_DISTINCT_NODES:
                want, occ_w = GSPF.place_gangs(node_off, rows, occ, req, off, quirks, E.POLICY_FIRST_FIT, node_table, lo2, hi2)
            else:       # any node on one node is a one-node gang there (G4)
                want, occ_w = GNF.place_gangs(node_off, rows, occ, req, off, quirks, E.POLICY_FIRST_FIT, node_table, lo2, hi2)
            assert np.array_equal(out, want) and np.array_equal(occ_g, occ_w), loc


@pytest.mark.parametrize("policy", POLICIES)
def test_n8d_committed_gangs_keep_their_locality(policy):
    """N8 (d): a committed one-node gang's members share a node, a committed distinct-node gang's members sit on distinct nodes."""
    rnd = random.Random(7500 + policy)
    for _ in range(150):
        node_off, rows, node_table, occ, req, off, quirks, policy, lo, hi, loc = _inputs(rnd, GSO.PER_GANG, policy)
        out, _, _ = GSF.place_gangs(node_off, rows, occ, req, off, policy, loc, quirks, node_table, lo, hi)
        for a, b in zip(off[:-1], off[1:]):
            alloc = np.flatnonzero(req["op"][a:b] == E.OP_ALLOC) + a
            if len(alloc) == 0 or not (out["status"][alloc] == E.ST_PLACED).all():
                continue
            nodes = np.searchsorted(node_off, out["gpu"][alloc], side="right") - 1
            if req["start"][alloc[0]] == E.GANG_ONE_NODE:
                assert len(set(nodes.tolist())) == 1
            elif req["start"][alloc[0]] == E.GANG_DISTINCT_NODES:
                assert len(set(nodes.tolist())) == len(alloc)


def test_n6_few_node_byte_refused_by_the_binding():
    """N6: the binding refuses a few-node locality on a node-scoring engine before it calls the library, as its other locality checks."""
    eng = E.Engine.__new__(E.Engine)
    eng.flags = E.FLAG_GANG_NODE_SCORE | E.FLAG_GANG_LOCALITY
    req = np.zeros(2, dtype=E.REQUEST_DTYPE)
    with pytest.raises(ValueError, match="few-node"):
        eng.place_gangs(req, [0, 1, 2], [E.GANG_ONE_NODE, E.GANG_FEW_NODES])
