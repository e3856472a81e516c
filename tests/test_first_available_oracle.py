"""Profile alternatives (ISL_FLAG_FIRST_AVAILABLE, include/islplace.h A1-A8) on the CPU: the brute force of
tests/first_available_fast.cpp against the composition of the unchanged checkers in tests/first_available_oracle.py on random clusters,
the hand-worked vectors, A4 and A5 (a) / (b) as properties, the run parsing at its edges, and the constants of the binding."""
import os
import re

import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import tables

import first_available_fast as F
import first_available_oracle as O

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG, E.POLICY_MOST_ALLOCATED,
            E.POLICY_LEAST_ALLOCATED]
TABLES3 = [tables.H100_80GB, tables.A30_24GB, tables.A100_40GB]


def random_cluster(rng, G, n_tables, fill=0.5):
    sizes = []
    while sum(sizes) < G:
        sizes.append(int(rng.choice([0, 1, 2, 4, 8])))
    sizes[-1] -= sum(sizes) - G
    node_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    names, rows = E.make_profile_tables(TABLES3[:n_tables])
    node_table = rng.integers(0, n_tables, len(sizes)).astype(np.uint8)
    occ = np.zeros(G, dtype=np.uint8)
    for x in range(8):
        occ |= ((rng.random(G) < fill).astype(np.uint8) << x)
    return node_off, rows, node_table, occ, len(names)


def random_pods(rng, n, n_names, G, max_run=4):
    out, pod = [], 0
    while len(out) < n:
        r = rng.random()
        if r < 0.08:
            out.append((int(rng.integers(0, G)), 0, E.OP_FREE, int(rng.integers(0, 8)), 1))
        elif r < 0.1:
            out.append((pod, 0, E.OP_NOOP, 0, 0))
        else:
            for _ in range(int(rng.integers(1, max_run + 1))):
                out.append((pod, int(rng.integers(0, n_names)) if rng.random() > 0.04 else E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0))
            pod += int(rng.random() > 0.1)
    return np.array(out[:n], dtype=E.REQUEST_DTYPE)


def _same(a, b):
    assert O.as_tuples(a[0]) == O.as_tuples(b[0])
    assert np.array_equal(a[1], b[1]) and a[2] == b[2]


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("policy", POLICIES)
def test_checkers_agree(policy, quirks):
    """The brute force and the composition of the unchanged checkers: whole inventory and a range that cuts nodes, 1 and 3 tables."""
    rng = np.random.default_rng(10 * policy + quirks)
    for n_tables in (1, 3):
        node_off, rows, node_table, occ, n = random_cluster(rng, 96, n_tables)
        req = random_pods(rng, 160, n, 96)
        _same(F.place(node_off, rows, occ, req, policy, quirks, node_table), O.place(node_off, rows, occ, req, policy, quirks, node_table))
        _same(F.place(node_off, rows, occ, req, policy, quirks, node_table, 13, 70),
              O.place(node_off, rows, occ, req, policy, quirks, node_table, 13, 70))


@pytest.mark.parametrize("case", O.kat_cases(), ids=lambda c: c["name"])
def test_kat(case):
    node_off, rows, node_table, occ, req, quirks, policy, (lo, hi) = O.case_inputs(case)
    for got in (F.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi),
                O.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)):
        assert O.as_tuples(got[0]) == O.expected(case)
        assert np.array_equal(got[1], O.runs(case["occ_after"]))


def test_kat_covers_the_issue():
    names = {c["name"] for c in O.kat_cases()}
    assert {"example_fixed", "example_ref_exact", "bad_profile_before_placed", "free_and_noop_split_handles", "right_to_left",
            "best_fit", "most_allocated", "least_allocated", "node_tables_choose"} <= names


@pytest.mark.parametrize("policy", POLICIES)
def test_a4_pods_of_one(policy):
    """A4: distinct adjacent handles, so the flagged rules equal isl_place_batch's (the brute force unflagged, and the unchanged
    checker through the composition), records, occupancy and placed count."""
    rng = np.random.default_rng(policy + 40)
    node_off, rows, node_table, occ, n = random_cluster(rng, 128, 3)
    req = random_pods(rng, 300, n, 128, max_run=1)
    alloc = np.flatnonzero(req["op"] == E.OP_ALLOC)
    req["handle"][alloc] = np.arange(len(alloc))
    flagged = F.place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table)
    _same(flagged, F.place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table, flagged=False))
    base = O._checker(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table, 0, 128)
    assert O.as_tuples(flagged[0]) == O.as_tuples(base[0]) and np.array_equal(flagged[1], base[1])


def _admits(rows2, node_off, node_table, occ, p, quirks, lo, hi):
    """Whether any GPU of [lo, hi) has a legal free start for profile p (its node's row)."""
    node_of = np.repeat(np.arange(len(node_off) - 1), np.diff(node_off.astype(np.int64)))
    for g in range(lo, hi):
        row = rows2[node_table[node_of[g]], p]
        for v in row["starts"][:row["n_starts"]]:
            v, z = int(v), int(row["size"])
            legal = z == 1 or ((not quirks & E.QUIRK_POW2_ONLY or z in (2, 4, 8)) and (v + z < 8 if quirks & E.QUIRK_STRICT_BOUND else v + z <= 8))
            if v < 8 and legal and not int(occ[g]) & (((1 << z) - 1) << v):
                return True
    return False


@pytest.mark.parametrize("policy", POLICIES)
def test_a5a_failed_alternative_fits_nowhere(policy):
    """A5 (a): replaying the records, every NO_CAPACITY alternative found no admitting GPU at its moment, every PLACED one the GPU it
    names admitted."""
    rng = np.random.default_rng(policy + 50)
    node_off, rows, node_table, occ, n = random_cluster(rng, 64, 3, fill=0.6)
    req = random_pods(rng, 200, n, 64)
    quirks = E.QUIRKS_REF_EXACT
    out, _, _ = F.place(node_off, rows, occ, req, policy, quirks, node_table)
    live = np.array(occ)
    for i in np.flatnonzero(req["op"] == E.OP_FREE):
        if out[i]["status"] == E.ST_FREED:
            live[int(req["handle"][i])] &= ~(((1 << int(req["size"][i])) - 1) << int(req["start"][i])) & 0xFF
    for i in np.flatnonzero(req["op"] == E.OP_ALLOC):
        st, p = int(out[i]["status"]), int(req["profile"][i])
        if st == E.ST_NO_CAPACITY:
            assert not _admits(rows, node_off, node_table, live, p, quirks, 0, 64)
        elif st == E.ST_PLACED:
            g = int(out[i]["gpu"])
            span = ((1 << int(out[i]["size"])) - 1) << int(out[i]["start"])
            assert not int(live[g]) & span
            live[g] |= span


@pytest.mark.parametrize("policy", POLICIES)
def test_a5b_chosen_only(policy):
    """A5 (b): each pod's chosen alternative alone, every other one a NOOP, through isl_place_batch's rules: same PLACED records, same
    occupancy."""
    rng = np.random.default_rng(policy + 60)
    node_off, rows, node_table, occ, n = random_cluster(rng, 96, 2)
    req = random_pods(rng, 250, n, 96)
    got, occ2, placed = F.place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table)
    alone, occ3, placed3 = F.place(node_off, rows, occ, O.chosen_only(req, got), policy, E.QUIRKS_FIXED, node_table, flagged=False)
    mask = got["status"] == E.ST_PLACED
    assert np.array_equal(alone["status"] == E.ST_PLACED, mask) and np.array_equal(alone[mask], got[mask])
    assert np.array_equal(occ2, occ3) and placed == placed3


@pytest.mark.parametrize("length", [16, 40])
def test_long_runs_and_repeated_profiles(length):
    """A run of 16 or 40 alternatives with repeated profiles: the first that fits is PLACED, every one after it ALT_SKIPPED, and a
    repeated profile after a failure fails again without changing anything."""
    rows = E.make_profiles(tables.H100_80GB)
    occ = np.array([0x7F, 0x3F], dtype=np.uint8)
    node_off = np.array([0, 1, 2], dtype=np.uint32)
    alts = ([5, 4, 3] * 20)[:length - 2] + [0, 0]          # 7g, 4g and 3g never fit; the first 1g does
    req = F.pods([alts, [0]])
    for policy in POLICIES:
        got, occ2, placed = F.place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED)
        _same((got, occ2, placed), O.place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED))
        st = list(got["status"])
        assert st[:length - 2] == [E.ST_NO_CAPACITY] * (length - 2)
        assert st[length - 2] == E.ST_PLACED and st[length - 1] == E.ST_ALT_SKIPPED
        assert got[length - 1]["size"] == 1 and got[length - 1]["gpu"] == E.GPU_NONE and got[length - 1]["start"] == E.START_NONE
        assert placed == 1 + (st[length] == E.ST_PLACED)


def test_equal_handles_split_by_free_or_noop():
    """A1: equal handles that are not adjacent are different pods."""
    assert list(O.pod_starts(np.array([(0, 1, E.OP_ALLOC, 0, 0), (0, 1, E.OP_ALLOC, 0, 0), (0, 0, E.OP_FREE, 0, 1),
                                       (0, 1, E.OP_ALLOC, 0, 0), (0, 0, E.OP_NOOP, 0, 0), (0, 1, E.OP_ALLOC, 0, 0),
                                       (1, 1, E.OP_ALLOC, 0, 0), (0, 1, E.OP_ALLOC, 0, 0), (0, 1, 7, 0, 0), (0, 1, E.OP_ALLOC, 0, 0)],
                                      dtype=E.REQUEST_DTYPE))) == [True, False, False, True, False, True, True, True, False, True]


def test_binding_mirrors_the_header():
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "islplace.h")).read()
    assert int(re.search(r"#define ISL_FLAG_FIRST_AVAILABLE (\d+)u", hdr).group(1)) == E.FLAG_FIRST_AVAILABLE == 1 << 15
    assert int(re.search(r"#define ISL_ST_ALT_SKIPPED\s+(\d+)u", hdr).group(1)) == E.ST_ALT_SKIPPED == 8
