"""The two restatements of node scoring (ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED): the hand-worked vectors of
tests/golden/kat_node_score.json through both, their agreement on random clusters, the one-node == first-fit consequence against the
CPU oracle, and the spreading property.  CPU only."""
import random

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import node_offsets

import node_score_fast as NF
import node_score_oracle as NO

POLICIES = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]
TABLE_NAMES = ["h100-80gb", "a30-24gb", "a100-40gb"]


@pytest.mark.parametrize("case", NO.kat_cases(), ids=lambda c: c["name"])
def test_kat_fast(case):
    node_off, rows, node_table, occ, req, quirks, policy, (lo, hi) = NO.case_inputs(case)
    out, after = NF.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
    assert [tuple(int(x) for x in r) for r in out] == NO.expected(case)
    assert np.array_equal(after, NO.runs(case["occ_after"]))


@pytest.mark.parametrize("case", NO.kat_cases(), ids=lambda c: c["name"])
def test_kat_cr(case):
    node_off, _rows, node_table, occ, _req, quirks, policy, (lo, hi) = NO.case_inputs(case)
    items = NO.items_from(node_off, occ, case["tables"], node_table)
    pods = NO.case_pods(case, items)
    got = NO.place_cr(items, pods, policy, quirks, lo, hi)
    assert NO.as_records(got) == NO.expected(case)
    assert np.array_equal(NO.occupancy(items), NO.runs(case["occ_after"]))


def test_kat_covers_what_it_claims():
    cases = NO.kat_cases()
    assert {c["policy"] for c in cases} == {"MOST_ALLOCATED", "LEAST_ALLOCATED"}
    assert {c["quirks"] for c in cases} == {"REF_EXACT", "FIXED"}
    assert any(len(c["tables"]) > 1 and "a30-24gb" in c["tables"] for c in cases)
    assert any("range" in c for c in cases)
    assert any(any(r[0] == "free" for r in c["requests"]) for c in cases)
    assert any(any(r[3] == "NO_CAPACITY" for r in c["records"]) for c in cases)
    assert any(any(a == b for a, b in zip(c["node_off"], c["node_off"][1:])) for c in cases)      # an empty node


def random_cluster(rnd, n_nodes, n_tables):
    """Unequal nodes (some empty), a random table per node, occupancy from random busy spans."""
    sizes = [0 if rnd.random() < 0.1 else rnd.choice([1, 1, 2, 3, 4, 7, 8, 16]) for _ in range(n_nodes)]
    if sum(sizes) == 0:
        sizes[0] = 1
    node_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    G = int(node_off[-1])
    occ = np.zeros(G, dtype=np.uint8)
    for g in range(G):
        full = rnd.random()
        for x in range(8):
            if rnd.random() < full * 0.9:
                occ[g] |= 1 << x
    node_table = np.array([rnd.randrange(n_tables) for _ in range(n_nodes)], dtype=np.uint8)
    return node_off, occ, node_table


def random_batch(rnd, names, occ, n):
    req = np.zeros(n, dtype=E.REQUEST_DTYPE)
    for i in range(n):
        x = rnd.random()
        if x < 0.12 and len(occ):
            g = rnd.randrange(len(occ))
            s = rnd.randrange(8)
            req[i] = (g, 0, E.OP_FREE, s, rnd.randint(1, 8 - s))
        elif x < 0.15:
            req[i] = (i, E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
        elif x < 0.17:
            req[i] = (i, 0, E.OP_NOOP, 0, 0)
        else:
            req[i] = (i, rnd.randrange(len(names)), E.OP_ALLOC, 0, 0)
    return req


@pytest.mark.parametrize("seed", range(40))
def test_restatements_agree(seed):
    """Random clusters with unequal and empty nodes, one or two tables, both quirk sets, ranges at unaligned bounds; FREEs of whole
    busy spans only, so that the CR side can name them as allocations."""
    rnd = random.Random(seed)
    n_tables = 1 + seed % 2
    table_names = TABLE_NAMES[:n_tables] if seed % 4 < 2 else ["a30-24gb", "h100-80gb"][:n_tables]
    names, rows = E.make_profile_tables([tables.TABLES[t] for t in table_names])
    node_off, occ, node_table = random_cluster(rnd, rnd.randint(1, 24), n_tables)
    G = int(node_off[-1])
    quirks = rnd.choice([E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
    policy = POLICIES[seed % 2]
    lo, hi = (0, G) if seed % 3 == 0 else sorted(rnd.sample(range(G + 1), 2)) if G > 1 else (0, G)
    req = random_batch(rnd, names, occ, rnd.randint(1, 60))
    items = NO.items_from(node_off, occ, table_names, node_table)
    # a FREE on the flat side must name exactly the span the CR side releases: make every FREE's span an allocation of its own
    pods = []
    for i, r in enumerate(req):
        if r["op"] == E.OP_FREE:
            g, s, z = int(r["handle"]), int(r["start"]), int(r["size"])
            n = int(np.searchsorted(node_off, g, side="right")) - 1
            spec = items[n]["spec"]
            if all(int(occ[g]) >> x & 1 and ("p%d-%d" % (g, x)) in spec["prepared"] for x in range(s, s + z)):
                for x in range(s, s + z):
                    del spec["prepared"]["p%d-%d" % (g, x)]
                spec["allocations"]["old-%d" % i] = {"gpuUUID": "GPU-%07d" % g, "start": s, "size": z, "allocationStatus": "created"}
                pods.append({"op": "free", "uid": "old-%d" % i})
                continue
            req[i]["op"] = E.OP_NOOP
        if req[i]["op"] == E.OP_ALLOC:
            name = names[r["profile"]] if r["profile"] < len(names) else "unknown"
            pods.append({"op": "alloc", "profile": name, "uid": "pod-%d" % i})
        else:
            pods.append({"op": "noop"})
    out, after = NF.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
    got = NO.place_cr(items, pods, policy, quirks, lo, hi, names)
    for i, r in enumerate(req):
        if req[i]["op"] == E.OP_NOOP:
            assert int(out[i]["status"]) == E.ST_NOOP
            continue
        assert tuple(int(x) for x in out[i]) == NO.as_records([got[i]])[0], (i, r)
    assert np.array_equal(after, NO.occupancy(items))


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_one_node_is_first_fit(policy, quirks):
    """On an inventory of one node the only candidate is that node, and inside it the reference's own search decides."""
    rng = np.random.default_rng(policy * 10 + quirks)
    rnd = random.Random(quirks)
    node_off = np.array([0, 24], dtype=np.uint32)
    occ = (rng.integers(0, 256, 24) & rng.integers(0, 256, 24)).astype(np.uint8)
    rows = E.make_profiles(tables.H100_80GB)
    req = random_batch(rnd, [r[0] for r in tables.H100_80GB], occ, 200)
    out, after = NF.place(node_off, rows, occ, req, policy, quirks)
    ref = oracle.Fast(node_off, rows, quirks=quirks)
    ref.load(occ)
    assert np.array_equal(out, ref.place(req))
    assert np.array_equal(after, ref.occupancy())


@pytest.mark.parametrize("n_nodes", [1, 5, 64])
def test_least_allocated_spreads(n_nodes):
    """LeastAllocated on an empty cluster of equal 8-GPU nodes places the first n_nodes one-slice pods on n_nodes distinct nodes, in
    node order; MostAllocated puts them all on node 0."""
    node_off = node_offsets(n_nodes, 8)
    rows = E.make_profiles(tables.H100_80GB)
    req = np.zeros(n_nodes, dtype=E.REQUEST_DTYPE)
    req["op"] = E.OP_ALLOC
    out, _ = NF.place(node_off, rows, np.zeros(8 * n_nodes, dtype=np.uint8), req, E.POLICY_LEAST_ALLOCATED)
    assert (out["status"] == E.ST_PLACED).all()
    assert list(out["gpu"] // 8) == list(range(n_nodes)) and (out["start"] == 0).all()
    out, _ = NF.place(node_off, rows, np.zeros(8 * n_nodes, dtype=np.uint8), req, E.POLICY_MOST_ALLOCATED)
    assert (out["gpu"][:56] < 8).all()                  # node 0 takes 8 x 7 one-slice pods before any other node gets one
    assert list(out["start"][:7]) == list(range(min(7, n_nodes)))
