"""One-node gangs (k_ganglocal<one_node>) and distinct-node gangs (k_ganglocal<distinct_nodes>) at the limits of the profile-table ABI, of
the inventory and of their shared layout (gang_layout), on the H100.  Every call is compared with its brute force (tests/gang_node_fast.cpp,
tests/gang_spread_fast.cpp) — every record and the final occupancy — and its committed gangs are checked against the topology rule through
isl_gpu_to_node: one node per gang, or pairwise distinct nodes.  The inputs come from ``test_oracle_gang_topology_limits.py``, which pins
the checkers at these shapes and shows that every generator reaches its edge.

  fixtures     T16x8, T16mix-1/2 under quirk sets 0-3, T8tab with node tables, T16top, T16straddle; every policy; 4 096 / 4 097 GPUs
               of eight-GPU nodes, whole bytes, every gang shape
  calls        one-node pass 0 (perfect fits behind decoys, failures deepest on skipped nodes), profile 15 dead only after a failure
               at rank 0, MIN_FRAG scores of 121 and on both sides of 64, more than 510 gangs (the node-used tags wrap)
  2^20 GPUs    T8tab with node tables, every policy, the lower half full but for what the call's FREEs release; under right-to-left also
               the top partition [2^20 - 4 109, 2^20), which cuts a node
  layout       every gang_plan edge at the device's SM count and shared-memory opt-in, on both sides of the shared / global switch
"""
import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

from test_oracle_gang_topology_limits import (CASES, FIXTURES, KERNELS, LAYOUT_CASES, POLICIES, case_ids, dead15_call, gang_plan,
                                              layout_cases, lower_half_full, min_frag_call, pass0_call, pass1_call, small_gangs,
                                              wrap_call)
from test_oracle_request_major_limits import GANG_SHAPES, eight_gpu_nodes, gang_call, gang_offsets, node_tables_for, whole_bytes
from test_oracle_table_limits import t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu


def make_engine(kind, rows, policy, quirks, max_gpus=4097, max_batch=1 << 16):
    eng = E.Engine(max_gpus=max_gpus, max_batch=max_batch, policy=policy, quirks=quirks, flags=KERNELS[kind][0])
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    return eng


def load(eng, node_off, occ, node_table):
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)


def device():
    import torch
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


def check(eng, kind, rows, node_off, node_table, occ, req, off, quirks, policy, part=None, what=""):
    """Load the inventory (and the partition), place the call, compare with the brute force and check the topology rule."""
    G = int(node_off[-1])
    lo, hi = part or (0, G)
    load(eng, node_off, occ, node_table)
    if part:
        eng.set_partition(lo, hi)
    want, occ_want = KERNELS[kind][1](node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
    got = eng.place_gangs(req, off)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), occ_want), what
    for a, b in zip(off[:-1], off[1:]):
        sel = (got["status"][a:b] == E.ST_PLACED) & (req["op"][a:b] == E.OP_ALLOC)
        nodes = [eng.gpu_to_node(int(g)) for g in got["gpu"][a:b][sel]]
        if kind == "one_node":
            assert len(set(nodes)) <= 1, (what, a, b, nodes)
        else:
            assert len(set(nodes)) == len(nodes), (what, a, b, nodes)
    return got


# ---- every fixture, quirk set and policy at 4 096 / 4 097 GPUs ------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=case_ids(CASES))
@pytest.mark.parametrize("kind", list(KERNELS))
def test_fixtures(kind, name, quirks, policy):
    rows = FIXTURES[name]()
    rng = W.SplitMix64(9000 + 10 * policy + quirks + len(name) + 100 * len(kind))
    n = 300 if policy == E.POLICY_MIN_FRAG else 1000
    eng = make_engine(kind, rows, policy, quirks)
    outcomes = set()
    for G in (4096, 4097):
        node_off = eight_gpu_nodes(G)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        for shape in GANG_SHAPES:
            occ = whole_bytes(rng, G, dense=True)
            got = check(eng, kind, rows, node_off, node_table, occ, gang_call(rng, G, rows.shape[-1], n), gang_offsets(rng, shape, n),
                        quirks, policy, what=(G, shape))
            outcomes |= set(np.unique(got["status"]).tolist())
    eng.close()
    assert {E.ST_PLACED, E.ST_GANG_ABORTED} <= outcomes


# ---- the calls built for one edge each ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("kind", list(KERNELS))
def test_pass0_filter_calls(kind, policy):
    """The one-node pass 0 at its edges (free slices equal to the need, first and behind a decoy; the deepest failure on a skipped
    node), T8tab with absent rows and tables 0..7; the same calls on the distinct-node engine."""
    rows = t8tab()
    rng = W.SplitMix64(600 + policy)
    eng = make_engine(kind, rows, policy, E.QUIRKS_FIXED)
    for G in (4096, 4097):
        node_off, node_table, occ, req, off, _pairs = pass0_call(rng, policy, G)
        check(eng, kind, rows, node_off, node_table, occ, req, off, E.QUIRKS_FIXED, policy, what=("pass 0", G))
    node_off, node_table, occ, req, off, _pairs = pass1_call(W.SplitMix64(700 + policy), policy)
    got = check(eng, kind, rows, node_off, node_table, occ, req, off, E.QUIRKS_FIXED, policy, what="pass 1")
    if kind == "one_node":
        assert got["status"].reshape(-1, 3)[:, 2].tolist() == [E.ST_NO_CAPACITY] * 3
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", [("t16x8", E.QUIRKS_REF_EXACT), ("t8tab", E.QUIRKS_FIXED), ("t16top", E.QUIRKS_FIXED)])
@pytest.mark.parametrize("kind", list(KERNELS))
def test_profile_15_dead_only_after_rank_0(kind, name, quirks, policy):
    """The distinct-node dead mask: profile 15 failing behind the exclusion (rank >= 1) stays live, failing at rank 0 is dead."""
    rows = FIXTURES[name]()
    rng = W.SplitMix64(1500 + policy + len(name))
    node_off, node_table, occ, req, off, want = dead15_call(rng, rows, quirks)
    eng = make_engine(kind, rows, policy, quirks)
    got = check(eng, kind, rows, node_off, node_table, occ, req, off, quirks, policy)
    if kind == "distinct_nodes":
        assert [got["status"][a:b].tolist() for a, b in zip(off[:-1], off[1:])] == want
    eng.close()


@pytest.mark.parametrize("name", ["t16top", "t16straddle"])
@pytest.mark.parametrize("kind", list(KERNELS))
def test_min_frag_scores_above_63(kind, name):
    """ISL_POLICY_MIN_FRAG member keys with the largest score (121, T16top) and with scores on both sides of 64 (T16straddle)."""
    rng = W.SplitMix64(121)
    rows, node_off, occ, req, off = min_frag_call(rng, name)
    eng = make_engine(kind, rows, E.POLICY_MIN_FRAG, E.QUIRKS_FIXED)
    got = check(eng, kind, rows, node_off, None, occ, req, off, E.QUIRKS_FIXED, E.POLICY_MIN_FRAG)
    assert (got["status"][req["profile"] == 15] == E.ST_PLACED).any()
    eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_MIN_FRAG])
@pytest.mark.parametrize("kind", list(KERNELS))
def test_tags_wrap_with_profile_15_live(kind, policy):
    rng = W.SplitMix64(255)
    rows, node_off, occ, req, off = wrap_call(rng, 1800 if policy == E.POLICY_FIRST_FIT else 900)
    eng = make_engine(kind, rows, policy, E.QUIRKS_REF_EXACT)
    got = check(eng, kind, rows, node_off, None, occ, req, off, E.QUIRKS_REF_EXACT, policy)
    gang = np.searchsorted(off, np.arange(len(req)), side="right") - 1
    assert len(off) - 1 > 255 and ((req["profile"] == 15) & (got["status"] == E.ST_PLACED) & (gang >= 255)).any()
    eng.close()


# ---- 2^20 GPUs ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("kind", list(KERNELS))
def test_2_20_gpus(kind, policy):
    """T8tab on 2^20 GPUs with node tables: 132 CTAs of about 7 944 GPUs; placements at GPU indices with bit 19 set.  Under
    right-to-left the same engine then takes the top partition [2^20 - 4 109, 2^20), which cuts a node (flip and storage_range)."""
    G = 1 << 20
    rng = W.SplitMix64(G + policy + len(kind))
    rows, node_off, node_table, occ, req, off = lower_half_full(rng, G, 120 if policy == E.POLICY_MIN_FRAG else 200)
    eng = make_engine(kind, rows, policy, E.QUIRKS_FIXED, max_gpus=G)
    got = check(eng, kind, rows, node_off, node_table, occ, req, off, E.QUIRKS_FIXED, policy, what="2^20")
    placed = (got["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)
    assert (got["gpu"][placed] >= G // 2).any() and (got["status"] == E.ST_GANG_ABORTED).any()
    if policy == E.POLICY_RIGHT_TO_LEFT:
        lo = G - 4096 - 13
        occ = whole_bytes(rng, G)
        req = gang_call(rng, G, 16, 400)
        top = np.flatnonzero(req["op"] == E.OP_FREE)[::2]
        req["handle"][top] = lo + (req["handle"][top] % np.uint32(G - lo))     # half the FREEs inside the partition
        got = check(eng, kind, rows, node_off, node_table, occ, req, small_gangs(rng, 400), E.QUIRKS_FIXED, policy, part=(lo, G),
                    what="top partition")
        assert (got["status"] == E.ST_PLACED).any() and (got["gpu"][got["status"] == E.ST_PLACED] >= lo).all()
    eng.close()


# ---- the layout edges on this device --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", LAYOUT_CASES)
@pytest.mark.parametrize("kind", list(KERNELS))
def test_layout_edges(kind, case):
    """Every gang_plan edge built from this device's SM count and shared-memory opt-in; the kernels' static shared memory is under
    1 KiB, so gang_plan's side of the shared / global switch holds for every static size up to that."""
    sms, optin = device()
    node_off, lo, hi, edge = layout_cases(sms, optin)[case]
    for static in (0, 1024):
        assert edge(gang_plan(node_off, lo, hi, sms, optin - static)), (case, static)
    i = LAYOUT_CASES.index(case)
    policy = (E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG)[i % 3]
    rows = t8tab()
    rng = W.SplitMix64(80 + i)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    occ = whole_bytes(rng, G)
    n = 200 if policy == E.POLICY_MIN_FRAG else 400
    eng = make_engine(kind, rows, policy, E.QUIRKS_FIXED, max_gpus=max(4097, G))
    part = None if (lo, hi) == (0, G) else (lo, hi)
    got = check(eng, kind, rows, node_off, node_table, occ, gang_call(rng, G, 16, n), small_gangs(rng, n), E.QUIRKS_FIXED, policy,
                part, what=case)
    assert (got["status"] == E.ST_PLACED).any()
    eng.close()
