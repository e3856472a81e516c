"""Gang preemption's two CPU restatements (tests/gang_preempt_fast.cpp on flat bytes, tests/gang_preempt_oracle.py on top of the unchanged
preempt_fast): the hand-worked vectors, agreement on random clusters, and the consequences P6 (a), (b), (d), (e) and P1's refusals
(include/islplace.h)."""
import random

import numpy as np
import pytest

from instaslice_b200 import engine as E

import gang_locality_oracle as GLO
import gang_preempt_fast as GF
import gang_preempt_oracle as GO
import preempt_fast as PF

LOCS = [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GO.PER_GANG]


@pytest.mark.parametrize("checker", [GF.preempt, GO.preempt], ids=["fast", "oracle"])
@pytest.mark.parametrize("case", GO.kat_cases(), ids=lambda c: c["name"])
def test_kat(case, checker):
    rc, out, evict = GO.run(checker, GO.case_inputs(case))
    recs, ev = GO.expected(case)
    assert rc == E.OK
    assert [tuple(int(x) for x in r) for r in out] == recs
    assert [[int(k) for k in row if k != E.GPU_NONE] for row in evict] == ev


def test_kat_covers_the_issue_examples():
    names = {c["name"] for c in GO.kat_cases()}
    assert {"p8_small_first_aborts", "p8_large_first_commits", "one_node_two_cheap_victims", "scan_tie_first_fit",
            "scan_tie_right_to_left", "one_node_failure_depth", "distinct_evicts_on_second_node", "mixed_localities", "two_node_tables",
            "noop_members"} <= names


@pytest.mark.parametrize("loc", LOCS)
def test_checkers_agree(loc):
    rnd = random.Random(11 + loc)
    for it in range(150):
        _n, rows = GO.random_rows(rnd)
        inputs = GO.random_case(rnd, rnd.randint(1, 30), rnd.randint(1, 16), rows, max_gang=6, locality=loc)
        a, b = GO.run(GF.preempt, inputs), GO.run(GO.preempt, inputs)
        assert a[0] == b[0] == E.OK
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])


@pytest.mark.parametrize("loc", LOCS)
def test_gangs_of_one_equal_preempt(loc):
    """P6 (a): with every handle distinct, a flagged call equals isl_preempt (preempt_fast) under every policy, quirks and partition."""
    rnd = random.Random(21 + loc)
    for it in range(150):
        _n, rows = GO.random_rows(rnd)
        inputs = list(GO.random_case(rnd, rnd.randint(1, 30), rnd.randint(1, 16), rows, max_gang=1, locality=loc))
        inputs[4] = inputs[4].copy()
        inputs[4]["handle"] = np.arange(len(inputs[4]))
        node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, _ = inputs
        rc, out, evict = GO.run(GF.preempt, tuple(inputs))
        want = PF.preempt(node_off, rows, occ, req, prio, vic, quirks=quirks, policy=policy, node_table=node_table, lo=lo, hi=hi)
        assert rc == want[0] == E.OK
        assert np.array_equal(out, want[1]) and np.array_equal(evict, want[2])


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
@pytest.mark.parametrize("loc", LOCS)
def test_no_victims_equal_place_gangs(policy, loc):
    """P6 (b): with no victim below its gang's priority, the records of isl_place_gangs (the existing gang checkers, dispatched per
    locality by gang_locality_oracle over gang_oracle, gang_node_fast and gang_spread_fast)."""
    rnd = random.Random(31 + loc + 7 * policy)
    for it in range(80):
        _n, rows = GO.random_rows(rnd)
        node_off, rows, node_table, occ, req, prio, vic, quirks, _p, lo, hi, _ = GO.random_case(rnd, rnd.randint(1, 24), rnd.randint(1, 16),
                                                                                             rows, max_gang=5, locality=loc, policy=policy)
        req = req.copy()
        if loc != GO.PER_GANG:
            req["start"] = loc
        prio = prio.copy()
        if it % 2:
            vic = vic[:0]
        else:
            prio[:] = 0
        rc, out, evict = GO.run(GF.preempt, (node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc))
        bounds = GO.gang_bounds(req)
        want, _occ = GLO.fast_gangs_locality(node_off, rows, occ, req, [a for a, _ in bounds] + [len(req)], quirks, policy, node_table,
                                             lo, hi)
        assert rc == E.OK and np.array_equal(out, want)
        assert (evict == E.GPU_NONE).all()


def _node_of(node_off, g):
    return int(np.searchsorted(node_off, g, side="right")) - 1


@pytest.mark.parametrize("loc", LOCS)
def test_committed_gangs_fit(loc):
    """P6 (d): with the victims of a committed gang and of every committed gang before it removed, its spans are free and disjoint; a
    one-node gang shares one node, a distinct-node gang's members sit on distinct nodes."""
    rnd = random.Random(41 + loc)
    for it in range(120):
        _n, rows = GO.random_rows(rnd)
        node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc_ = GO.random_case(rnd, rnd.randint(1, 24), 16, rows,
                                                                                                     max_gang=5, locality=loc)
        rc, out, evict = GO.run(GF.preempt, (node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc_))
        assert rc == E.OK
        cur = occ.copy()
        for a, b in GO.gang_bounds(req):
            al = [r for r in range(a, b) if req[r]["op"] == E.OP_ALLOC]
            if not al or out[al[0]]["status"] != E.ST_PLACED:
                assert all(out[r]["status"] != E.ST_PLACED for r in al)
                assert (evict[a:b] == E.GPU_NONE).all()
                continue
            for k in {int(k) for k in evict[a:b].ravel() if k != E.GPU_NONE}:
                cur[vic[k]["gpu"]] &= ~(((1 << int(vic[k]["size"])) - 1) << int(vic[k]["start"])) & 0xFF
            for r in al:
                span = ((1 << int(out[r]["size"])) - 1) << int(out[r]["start"])
                g = int(out[r]["gpu"])
                assert lo <= g < hi and cur[g] & span == 0
                cur[g] |= span
            nodes = [_node_of(node_off, int(out[r]["gpu"])) for r in al]
            gloc = int(req[al[0]]["start"]) if loc == GO.PER_GANG else loc
            if gloc == E.GANG_ONE_NODE:
                assert len(set(nodes)) == 1
            if gloc == E.GANG_DISTINCT_NODES:
                assert len(set(nodes)) == len(nodes)


def test_any_node_equals_gangs_one_at_a_time():
    """P6 (e): under any-node locality a call equals its gangs run one at a time through isl_preempt (preempt_fast), each gang's
    evictions and spans applied when every member was placed and dropped otherwise."""
    rnd = random.Random(51)
    for it in range(150):
        _n, rows = GO.random_rows(rnd)
        node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, _ = GO.random_case(rnd, rnd.randint(1, 24), 16, rows,
                                                                                                  max_gang=5, locality=0)
        rc, out, evict = GO.run(GF.preempt, (node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, 0))
        cur, alive = occ.copy(), np.ones(len(vic), dtype=bool)
        for a, b in GO.gang_bounds(req):
            idx = np.flatnonzero(alive)
            _rc, o, ev = PF.preempt(node_off, rows, cur, req[a:b], prio[a:b], vic[idx], quirks=quirks, policy=policy,
                                    node_table=node_table, lo=lo, hi=hi)
            alloc = req[a:b]["op"] == E.OP_ALLOC
            if (o["status"][alloc] == E.ST_PLACED).all():
                ev = np.where(ev == E.GPU_NONE, E.GPU_NONE, idx[np.minimum(ev, max(len(idx) - 1, 0))] if len(idx) else ev)
                assert np.array_equal(out[a:b], o) and np.array_equal(evict[a:b], ev)
                for k in ev[ev != E.GPU_NONE]:
                    alive[k] = False
                    cur[vic[k]["gpu"]] &= ~(((1 << int(vic[k]["size"])) - 1) << int(vic[k]["start"])) & 0xFF
                for rec in o[alloc]:
                    cur[rec["gpu"]] |= ((1 << int(rec["size"])) - 1) << int(rec["start"])
            else:
                assert not (out[a:b]["status"] == E.ST_PLACED).any() and (evict[a:b] == E.GPU_NONE).all()


def _one_gang(names_rows, starts, prios, handles=(0, 0)):
    names, rows = names_rows
    req = np.zeros(len(starts), dtype=E.REQUEST_DTYPE)
    req["handle"] = handles[:len(starts)]
    req["profile"] = 0
    req["start"] = starts
    return (np.array([0, 2], dtype=np.uint32), rows, None, np.zeros(2, dtype=np.uint8), req, np.array(prios, dtype=np.uint8),
            np.zeros(0, dtype=E.VICTIM_DTYPE), E.QUIRKS_REF_EXACT, E.POLICY_FIRST_FIT, 0, 2)


@pytest.mark.parametrize("checker", [GF.preempt, GO.preempt], ids=["fast", "oracle"])
def test_p1_einval(checker):
    """P1: two priorities in one gang; under per-gang locality two locality bytes, byte 2 (few nodes) or above 3; rule 3's FREE.  A
    NOOP member's bytes are not looked at, and the same bytes in different gangs are accepted."""
    nr = GO.random_rows(random.Random(1), 1)
    assert GO.run(checker, _one_gang(nr, [0, 0], [1, 2]) + (0,))[0] == E.EINVAL
    for s in ([0, 1], [1, 3], [2, 2], [4, 4], [9, 9]):
        assert GO.run(checker, _one_gang(nr, s, [1, 1]) + (GO.PER_GANG,))[0] == E.EINVAL
    assert GO.run(checker, _one_gang(nr, [2, 2], [1, 1]) + (0,))[0] == E.OK              # the byte names nothing without the flag
    assert GO.run(checker, _one_gang(nr, [0, 1], [1, 2], (0, 1)) + (GO.PER_GANG,))[0] == E.OK
    inp = list(_one_gang(nr, [2, 0], [9, 1]))
    inp[4] = inp[4].copy()
    inp[4]["op"][0] = E.OP_NOOP
    assert GO.run(checker, tuple(inp) + (GO.PER_GANG,))[0] == E.OK
    inp[4]["op"][0] = E.OP_FREE
    assert GO.run(checker, tuple(inp) + (GO.PER_GANG,))[0] == E.EINVAL


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT])
def test_node_index_above_2_20(policy):
    """Empty nodes are node indices: both checkers send the one-node gang to node 2^20 + 1 (GPU 2), whole."""
    for checker in (GF.preempt, GO.preempt):
        rc, out, evict = GO.run(checker, GO.node_index_case(policy))
        assert rc == E.OK
        assert out["status"].tolist() == [E.ST_PLACED, E.ST_PLACED] and out["gpu"].tolist() == [2, 2]
        assert out["start"].tolist() == [0, 1] and (evict == E.GPU_NONE).all()
