"""Gangs (k_bestfit<.., kGang = true>), preemption (k_victim_map + k_preempt) and node scoring (k_nodefit) at the limits of the
profile-table ABI and of the inventory, on the H100.  Every call is compared byte for byte with its CPU checker — records, evict rows
and final occupancy — on the fixtures of ``test_oracle_table_limits.py`` and the generators of ``test_oracle_request_major_limits.py``
(which pins the checkers at these shapes and checks that the generators reach their edges).

  gangs         T16x8, T16mix-1/2 under quirk sets 0-3, T8tab with node tables; every policy; gangs of one, mixed, one straddling
                32-request blocks, one that is the whole call; G = 4096 / 4097 (class bitmaps in shared / global memory); profile 15
                dying inside an aborted gang and placed after it; 2^20 GPUs; gangs of one == isl_place_batch on T8tab
  preemption    T16x8 (position 7 of 8-start rows), T16mix-2 under FIXED quirks (sizes 3, 5, 6, 7), T8tab with node tables; every
                policy at the G where the last CTA owns one GPU; 2^20 GPUs, right-to-left, and the top partition [2^20 - 1000, 2^20) where
                eight victims of priority 254 leave at once (the largest sum the key holds)
  node scoring  T16x8, T16mix-2 (width 10), T8tab (8 tables of several widths, names a table lacks); both policies and quirk sets;
                2 048 / 2 049 nodes (score trees in shared / global memory) and a range that cuts nodes; 2^20 nodes with empty ones
                (five full tree levels); 2^20 + 1 nodes refused with ISL_ERANGE, the previous inventory kept
"""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

import gang_oracle as GO
import node_score_fast as NF
import preempt_fast as PF
from test_oracle_request_major_limits import (FIXTURES, GANG_SHAPES, QUIRKS2, eight_gpu_nodes, gang_call, gang_offsets, gang_sizes,
                                              node_tables_for, p15_call, preempt_state, preemptors_for, row_positions,
                                              scoring_nodes, sm_limit_gpus, top_nodes, top_partition_case, whole_bytes, winner_stats)
from test_oracle_table_limits import t16x8, t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
SCORING = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]


def make_engine(rows, policy, quirks, max_gpus=4097, max_batch=1 << 16):
    eng = E.Engine(max_gpus=max_gpus, max_batch=max_batch, policy=policy, quirks=quirks)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    return eng


def load(eng, node_off, occ, node_table):
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def assert_same(got, want, what):
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])


# ---- gangs -----------------------------------------------------------------------------------------------------------------------
def check_gangs(eng, rows, node_off, node_table, occ, req, off, quirks, policy, what):
    ref = oracle.Fast(node_off, rows, quirks, policy, node_table=node_table)
    ref.load(occ)
    want = GO.fast_place_gangs(ref, req, off, gang_sizes(rows, node_table))
    load(eng, node_off, occ, node_table)
    got = eng.place_gangs(req, off)
    assert_same(got, want, what)
    assert np.array_equal(eng.read_occupancy(), ref.occupancy()), what
    return got


GANG_CASES = [("t16x8", E.QUIRKS_REF_EXACT)] + [(f, q) for f in ("t16mix1", "t16mix2") for q in (0, 1, 2, 3)] + [("t8tab", E.QUIRKS_FIXED)]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", GANG_CASES)
def test_gangs(name, quirks, policy):
    rows = FIXTURES[name]()
    rng = W.SplitMix64(5000 + 10 * policy + quirks + len(name))
    n = 300 if policy == E.POLICY_MIN_FRAG else 1500
    eng = make_engine(rows, policy, quirks)
    outcomes = set()
    for G in (4096, 4097):
        node_off = eight_gpu_nodes(G)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        for kind in GANG_SHAPES:
            occ = whole_bytes(rng, G, dense=True)           # dense: profiles run out and gangs abort
            got = check_gangs(eng, rows, node_off, node_table, occ, gang_call(rng, G, rows.shape[-1], n), gang_offsets(rng, kind, n),
                              quirks, policy, (G, kind))
            outcomes |= set(np.unique(got["status"]).tolist())
        # profile 15 dies inside an aborted gang (bit 15 of the saved dead mask) and is placed by the gangs after it
        occ, req, off = p15_call(rng, rows, node_off, node_table, quirks)
        got = check_gangs(eng, rows, node_off, node_table, occ, req, off, quirks, policy, (G, "p15"))
        outcomes |= set(np.unique(got["status"]).tolist())
        if name != "t16mix1" and name != "t16mix2":         # T16mix: no quirk set places profile 15
            assert got["status"][int(off[1]) - 1] == E.ST_NO_CAPACITY and got["status"][int(off[3]) - 1] == E.ST_PLACED
    eng.close()
    assert {E.ST_PLACED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY, E.ST_FREED, E.ST_NOOP} <= outcomes


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT])
def test_gangs_at_2_20_gpus(policy):
    """T8tab on 2^20 GPUs: the class bitmaps of 8 tables in global memory at kBfMaxGpus; the lower half full but for what the call's
    FREEs release, so that placements land at GPU indices with bit 19 set."""
    rows = t8tab()
    rng = W.SplitMix64(1 << 20)
    G = 1 << 20
    node_off = eight_gpu_nodes(G)
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    eng = make_engine(rows, policy, E.QUIRKS_FIXED, max_gpus=G)
    occ = whole_bytes(rng, G, dense=True)
    occ[: G // 2] = 0xFF
    n = 400
    got = check_gangs(eng, rows, node_off, node_table, occ, gang_call(rng, G, 16, n), gang_offsets(rng, "straddle", n), E.QUIRKS_FIXED,
                      policy, "2^20")
    placed = got["status"] == E.ST_PLACED
    assert (got["gpu"][placed] >= G // 2).any() and (got["status"] == E.ST_GANG_ABORTED).any()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_gangs_of_one_equal_place_batch_t8tab(policy):
    rows = t8tab()
    rng = W.SplitMix64(11 + policy)
    G = 4097
    node_off = eight_gpu_nodes(G)
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    occ = whole_bytes(rng, G)
    a, b = make_engine(rows, policy, E.QUIRKS_FIXED), make_engine(rows, policy, E.QUIRKS_FIXED)
    load(a, node_off, occ, node_table)
    load(b, node_off, occ, node_table)
    for _ in range(2):
        req = gang_call(rng, G, 16, 3000 if policy != E.POLICY_MIN_FRAG else 800)
        assert_same(a.place_gangs(req, np.arange(len(req) + 1)), b.place_batch(req), policy)
        assert np.array_equal(a.read_occupancy(), b.read_occupancy())
    a.close()
    b.close()


# ---- preemption -------------------------------------------------------------------------------------------------------------------
def check_preempt(rows, node_off, node_table, occ, vic, req, prio, quirks, policy, lo=0, hi=None):
    G = int(node_off[-1])
    hi = G if hi is None else hi
    eng = make_engine(rows, policy, quirks, max_gpus=max(4096, G), max_batch=4096)
    load(eng, node_off, occ, node_table)
    if (lo, hi) != (0, G):
        eng.set_partition(lo, hi)
    out, evict = eng.preempt(req, prio, vic)
    rc, want, want_ev = PF.preempt(node_off, rows, occ, req, prio, vic, quirks, policy, node_table, lo, hi)
    assert rc == E.OK
    assert_same(out, want, (policy, lo, hi))
    assert np.array_equal(evict, want_ev)
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()
    return out, evict


PREEMPT_FIXTURES = [("t16x8", E.QUIRKS_REF_EXACT), ("t16mix2", E.QUIRKS_FIXED), ("t8tab", E.QUIRKS_FIXED)]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", PREEMPT_FIXTURES)
def test_preempt_where_the_last_cta_owns_one_gpu(name, quirks, policy):
    rows = FIXTURES[name]()
    G = sm_limit_gpus(sm_count())
    rng = np.random.default_rng(G + 10 * policy + quirks + len(name))
    node_off = eight_gpu_nodes(G)
    node_table = t8tab_node_tables(W.SplitMix64(policy), len(node_off) - 1) if rows.ndim == 2 else None
    occ, vic, _kinds = preempt_state(rng, G)
    req, prio = preemptors_for(rng, rows, 96)
    out, evict = check_preempt(rows, node_off, node_table, occ, vic, req, prio, quirks, policy)
    st = winner_stats(vic, evict, out)
    assert any(s[2] == 8 for s in st)                                       # a size-8 victim leaves
    if name == "t16x8":
        assert 7 in row_positions(rows, np.zeros(G, np.uint8), req, out)    # the last position of an 8-start row wins
    if name == "t16mix2":
        assert any(s[0] == 8 for s in st)                                   # eight victims at once


@pytest.mark.parametrize("name,quirks,policy", [("t16x8", E.QUIRKS_REF_EXACT, E.POLICY_RIGHT_TO_LEFT),
                                                ("t8tab", E.QUIRKS_FIXED, E.POLICY_FIRST_FIT)])
def test_preempt_at_2_20_gpus(name, quirks, policy):
    """2^20 GPUs: shares of 7 944 GPUs per CTA on 132 SMs and GPU keys in the top bits of the 24-bit field."""
    rows = FIXTURES[name]()
    G = 1 << 20
    rng = np.random.default_rng(policy + len(name))
    node_off = eight_gpu_nodes(G)
    node_table = t8tab_node_tables(W.SplitMix64(3), len(node_off) - 1) if rows.ndim == 2 else None
    occ, vic, _kinds = preempt_state(rng, G)
    req, prio = preemptors_for(rng, rows, 12 if name == "t16x8" else 24)
    out, _evict = check_preempt(rows, node_off, node_table, occ, vic, req, prio, quirks, policy)
    assert (out["status"] == E.ST_PLACED).any()


def test_preempt_top_partition_evicts_eight_victims_of_priority_254():
    """The partition [2^20 - 1000, 2^20) of a 2^20-GPU inventory, T16mix-2 under FIXED quirks, best-fit engine: preemptors of the size-8
    profile at priority 255 run through every cheaper GPU and then take eight victims of priority 254 (sum 2 032)."""
    rows = FIXTURES["t16mix2"]()
    G = 1 << 20
    lo = G - 1000
    rng = np.random.default_rng(2032)
    node_off = eight_gpu_nodes(G)
    occ, vic, req, prio = top_partition_case(rng, rows, G, lo, 400)
    out, evict = check_preempt(rows, node_off, None, occ, vic, req, prio, E.QUIRKS_FIXED, E.POLICY_BEST_FIT, lo, G)
    st = winner_stats(vic, evict, out)
    assert (8, 2032, 1) in st and any(s[2] == 8 for s in st)


# ---- node scoring -----------------------------------------------------------------------------------------------------------------
def scoring_batch(rng, n, n_names, G):
    req = gang_call(rng, G, n_names, n)
    frees = req["op"] == E.OP_FREE                     # FREEs of one slice, some outside the inventory
    req["size"][frees] = 1
    return req


def check_scoring(eng, rows, node_off, node_table, occ, req, policy, quirks, lo=None, hi=None, what=""):
    G = int(node_off[-1])
    want, after = NF.place(node_off, rows, occ, req, policy, quirks, node_table, 0 if lo is None else lo, G if hi is None else hi)
    got = eng.place_batch(req) if lo is None else eng.place_batch_range(lo, hi, req)
    assert_same(got, want, what)
    assert np.array_equal(eng.read_occupancy(), after), what
    return got, after


NODE_CASES = [(f, q) for f in ("t16x8", "t16mix2", "t8tab") for q in QUIRKS2]


@pytest.mark.parametrize("policy", SCORING)
@pytest.mark.parametrize("name,quirks", NODE_CASES)
def test_node_scoring(name, quirks, policy):
    rows = FIXTURES[name]()
    rng = W.SplitMix64(7000 + 10 * policy + quirks + len(name))
    eng = make_engine(rows, policy, quirks, max_gpus=1 << 15)
    placed = 0
    for n_nodes in (2048, 2049):
        node_off = scoring_nodes(rng, n_nodes)
        G = int(node_off[-1])
        node_table = node_tables_for(rows, rng, n_nodes)
        occ = whole_bytes(rng, G)
        load(eng, node_off, occ, node_table)
        got, after = check_scoring(eng, rows, node_off, node_table, occ, scoring_batch(rng, 3000, rows.shape[-1], G), policy, quirks,
                                   what=n_nodes)
        placed += int((got["status"] == E.ST_PLACED).sum())
        # a range whose both ends cut a node of several GPUs
        big = np.flatnonzero(np.diff(node_off.astype(np.int64)) >= 3)
        lo, hi = int(node_off[big[2]]) + 1, int(node_off[big[-3] + 1]) - 1
        check_scoring(eng, rows, node_off, node_table, after, scoring_batch(rng, 2000, rows.shape[-1], G), policy, quirks, lo, hi,
                      (n_nodes, lo, hi))
    assert placed > 0
    eng.close()


@pytest.mark.parametrize("policy,name,quirks", [(E.POLICY_MOST_ALLOCATED, "t16x8", E.QUIRKS_REF_EXACT),
                                                (E.POLICY_LEAST_ALLOCATED, "t8tab", E.QUIRKS_FIXED)])
def test_node_scoring_at_2_20_nodes(policy, name, quirks):
    """The largest inventory a node-scoring engine accepts: 2^20 nodes of 0..1 GPUs, empty ones included — five full tree levels."""
    rows = FIXTURES[name]()
    rng = W.SplitMix64(1 << 20)
    node_off = top_nodes(rng)
    G = int(node_off[-1])
    node_table = node_tables_for(rows, rng, len(node_off) - 1)
    occ = whole_bytes(rng, G)
    eng = make_engine(rows, policy, quirks, max_gpus=1 << 20)
    load(eng, node_off, occ, node_table)
    got, _after = check_scoring(eng, rows, node_off, node_table, occ, scoring_batch(rng, 300, rows.shape[-1], G), policy, quirks,
                                what="2^20 nodes")
    assert (got["status"] == E.ST_PLACED).any()
    eng.close()


@pytest.mark.parametrize("policy", SCORING)
def test_more_than_2_20_nodes_refused(policy):
    """2^20 + 1 nodes (no more GPUs than max_gpus) get ISL_ERANGE on a node-scoring engine; its inventory, partition and snapshot stay
    and it places on them.  A first-fit engine takes the same inventory."""
    rows = t16x8()
    rng = W.SplitMix64(policy)
    node_off = scoring_nodes(rng, 300)
    G = int(node_off[-1])
    occ = whole_bytes(rng, G)
    eng = make_engine(rows, policy, E.QUIRKS_REF_EXACT, max_gpus=1 << 20)
    load(eng, node_off, occ, None)
    lo, hi = 5, G - 7
    eng.set_partition(lo, hi)
    eng.snapshot_occupancy()
    big = top_nodes(rng, 1)
    assert len(big) - 1 == (1 << 20) + 1 and int(big[-1]) <= 1 << 20
    with pytest.raises(E.EngineError) as err:
        eng.load_inventory(big, np.zeros(int(big[-1]), dtype=np.uint8))
    assert err.value.code == E.ERANGE
    assert eng.num_gpus == G and np.array_equal(eng.read_occupancy(), occ)
    req = scoring_batch(rng, 2000, len(rows), G)
    want, after = NF.place(node_off, rows, occ, req, policy, E.QUIRKS_REF_EXACT, None, lo, hi)     # the partition is still in force
    assert_same(eng.place_batch(req), want, "after the refusal")
    assert np.array_equal(eng.read_occupancy(), after)
    eng.restore_occupancy()                                                 # the snapshot survived
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()
    ff = make_engine(rows, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT, max_gpus=1 << 20)
    ff.load_inventory(big, np.zeros(int(big[-1]), dtype=np.uint8))
    assert ff.num_gpus == int(big[-1])
    ff.close()
