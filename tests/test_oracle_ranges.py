"""The CPU restatement of isl_place_batch_range (``range_oracle.py``) pinned without a device: a hand-derived known answer, the whole
range against ``oracle.Fast``, the all-nodes composition against ``oracle.Faithful(all_nodes=True)``, and op values outside
ALLOC / FREE / NOOP in both oracles."""
import json
import os

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W

from range_oracle import OP_UNKNOWN, RangeFast, mixed_requests, place_range

HERE = os.path.dirname(os.path.abspath(__file__))
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]


def records(a):
    return [tuple(int(x) for x in r) for r in a]


def kat():
    with open(os.path.join(HERE, "golden", "kat_range.json")) as f:
        k = json.load(f)
    req = np.array([tuple(r) for r in k["requests"]], dtype=E.REQUEST_DTYPE)
    return k, req


def test_kat():
    k, req = kat()
    rows = E.make_profiles(tables.A100_40GB)
    ref = RangeFast(k["node_off"], rows, k["occ_before"], k["lo"], k["hi"])
    assert records(ref.place(req)) == [tuple(r) for r in k["records"]]
    assert ref.occupancy().tolist() == k["occ_after"]
    got, occ = place_range(k["node_off"], rows, k["occ_before"], k["lo"], k["hi"], req)
    assert records(got) == [tuple(r) for r in k["records"]] and occ.tolist() == k["occ_after"]


def test_unplaced_size_is_the_whole_inventory_default():
    """1g.10gb is 2 slices on an A100-40GB and 1 on an H100-80GB.  Node 0 (A100) is the first node with the name, so an unplaced
    1g.10gb reports 2 even when the range is node 1 (H100) alone."""
    names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB])
    p = names.index("1g.10gb")
    node_off, node_table = [0, 1, 2], np.array([0, 1], dtype=np.uint8)
    req = W.alloc_requests(np.array([p], dtype=np.uint8))
    got, occ = place_range(node_off, rows, [0x00, 0xFF], 1, 2, req, node_table=node_table)
    assert records(got) == [(E.GPU_NONE, 9, 2, E.ST_NO_CAPACITY)] and occ.tolist() == [0x00, 0xFF]
    got, occ = place_range(node_off, rows, [0x00, 0x00], 1, 2, req, node_table=node_table)
    assert records(got) == [(1, 0, 1, E.ST_PLACED)] and occ.tolist() == [0x00, 0x01]


def test_unknown_op_is_noop_in_both_oracles():
    """An op value the engine does not know gets a NOOP record (not the caller's untouched buffer, which reads as PLACED on GPU 0)."""
    rows = E.make_profiles(tables.A100_40GB)
    node_off, occ = W.node_offsets(2, 1), np.array([0x00, 0x0F], dtype=np.uint8)
    req = np.array([(0, 0, OP_UNKNOWN, 0, 0), (1, 0, 200, 0, 4), (0, 0, E.OP_ALLOC, 0, 0)], dtype=E.REQUEST_DTYPE)
    want = [(E.GPU_NONE, 9, 0, E.ST_NOOP), (E.GPU_NONE, 9, 0, E.ST_NOOP), (0, 0, 1, E.ST_PLACED)]
    fast = oracle.Fast(node_off, rows)
    fast.load(occ)
    assert records(fast.place(req)) == want and fast.occupancy().tolist() == [0x01, 0x0F]
    f = oracle.Faithful(node_off, rows)
    f.load_occupancy_as_dangling(occ)
    assert records(f.place(req)) == want and f.occupancy().tolist() == [0x01, 0x0F]


def cluster(rng, n_tables, n_nodes, gpn=4):
    node_off = W.node_offsets(n_nodes, gpn)
    if n_tables == 1:
        rows = E.make_profiles(tables.H100_80GB)
        return node_off, rows, None, len(rows)
    names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
    return node_off, rows, (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8), len(names)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_whole_range_is_fast(policy, quirks, n_tables):
    """[0, G) is byte-identical to oracle.Fast on the same requests: records and occupancy."""
    rng = W.SplitMix64(31 * policy + 7 * quirks + n_tables)
    node_off, rows, node_table, n_names = cluster(rng, n_tables, 75)
    G = int(node_off[-1])
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    fast = oracle.Fast(node_off, rows, quirks, policy, node_table=node_table)
    fast.load(occ)
    for n in (5, 40, 600):
        req = mixed_requests(rng, occ, 0, G, n_names, n)
        got, occ = place_range(node_off, rows, occ, 0, G, req, quirks, policy, node_table)
        assert np.array_equal(got, fast.place(req)), n
        assert np.array_equal(occ, fast.occupancy()), n


@pytest.mark.parametrize("seed", range(4))
def test_all_nodes_is_faithful(seed):
    """ISL_FLAG_ALL_NODES restated as one restricted call per node == the reference's node loop without its `break`, FREEs included
    (each one names a busy run of slices, which is what the structure-for-structure oracle can release)."""
    rng = W.SplitMix64(500 + seed)
    n_nodes, gpn = 6 + seed, 1 + seed
    node_off = W.node_offsets(n_nodes, gpn)
    G = int(node_off[-1])
    rows = E.make_profiles(tables.A100_40GB)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    f = oracle.Faithful(node_off, rows)
    f.load_occupancy_as_dangling(occ)
    runs = []                   # the dangling runs the structure oracle holds: a FREE must name one exactly
    for g in range(G):
        b, s = int(occ[g]), 0
        while s < 8:
            e = s
            while e < 8 and (b >> e) & 1:
                e += 1
            if e > s:
                runs.append((g, s, e - s))
            s = e + 1
    runs = [runs[int(i)] for i in np.argsort(rng.next(len(runs)))]      # shuffled; each is freed once
    for rep in range(3):
        req = mixed_requests(rng, occ, 0, G, len(rows), 60)
        valid = (req["op"] == E.OP_FREE) & (req["handle"] < G) & (req["size"] > 0) & (req["start"].astype(int) + req["size"] <= 8)
        for i in np.flatnonzero(valid):
            if runs:
                g, s, z = runs.pop()
                req[i] = (g, 0, E.OP_FREE, s, z)
            else:
                req["op"][i] = E.OP_NOOP
        got, occ = place_range(node_off, rows, occ, 0, G, req, all_nodes=True)
        want = f.place(req, all_nodes=True)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (rep, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
        assert np.array_equal(occ, f.occupancy()), rep


@pytest.mark.parametrize("policy", POLICIES)
def test_range_leaves_the_outside_alone(policy):
    """Any range, any policy: bytes outside [lo, hi) never change, every placement lands inside, and an outside FREE is FREED."""
    rng = W.SplitMix64(90 + policy)
    node_off, rows, node_table, n_names = cluster(rng, 3, 40, 3)
    G = int(node_off[-1])
    occ = (rng.next(G) & np.uint64(0x3F)).astype(np.uint8)
    for lo, hi in [(0, 0), (5, 5), (1, 2), (7, 31), (0, G), (G - 1, G)]:
        req = mixed_requests(rng, occ, lo, hi, n_names, 50)
        got, after = place_range(node_off, rows, occ, lo, hi, req, policy=policy, node_table=node_table)
        assert np.array_equal(np.r_[after[:lo], after[hi:]], np.r_[occ[:lo], occ[hi:]]), (lo, hi)
        placed = got[got["status"] == E.ST_PLACED]
        assert ((placed["gpu"] >= lo) & (placed["gpu"] < hi)).all(), (lo, hi)
        out_free = (req["op"] == E.OP_FREE) & ((req["handle"] < lo) | (req["handle"] >= hi)) & (req["handle"] < G) & (req["size"] > 0) & \
                   (req["start"].astype(int) + req["size"] <= 8)
        assert (got["status"][out_free] == E.ST_FREED).all(), (lo, hi)
        occ = after
