"""Profile alternatives (ISL_FLAG_FIRST_AVAILABLE, include/islplace.h A1-A8) at the limits of the ABI on the H100: k_bestfit<.., kAlt>
(FIRST_FIT, BEST_FIT, RIGHT_TO_LEFT, MIN_FRAG; one table and several) and k_nodefit<true> (MOST_ / LEAST_ALLOCATED) on the generators of
``test_oracle_first_available_limits.py``, which pins the brute force at these shapes and shows that every generator reaches its edge.

Every call is compared with tests/first_available_fast.cpp (with its score memo) byte for byte: every record, the whole occupancy after the call, and the deltas
of the counters — ``requests``, ``placed``, ``no_capacity`` (the ALLOCs of a known profile that were not placed, ALT_SKIPPED ones
included), ``kernel_launches`` (k_prepare + the request-major kernel, 2 per batch; isl_what_if 2 more for its capacities); ``freed`` and
``batches`` equal those of an engine without the flag given the same calls.

  fixtures      T16x8 (REF_EXACT), T16mix-1/2 under quirk sets 0-3, T8tab (FIXED) with node tables, every policy: 4 096 and 4 097 GPUs
                of eight-GPU nodes for k_bestfit, 2 048 and 2 049 ragged nodes with empty ones for k_nodefit, and a range that cuts nodes
                at both ends; T16top and T16straddle under best-fit and min-frag
  edges         long runs over up to four 32-request blocks, pods opening at lane 0 and lane 31, ops 3..255, handles that differ in bit
                16 or 31 only, 0xFFFFFFFF, profile bytes >= the name count; profile 15 dead within a launch and alive in the next, through
                two isl_place_batch calls and one isl_place_stream
  2^20 GPUs     T8tab with node tables, the lower half full, every policy, through isl_place_batch, isl_place_batch_range and a partition;
                T16x8 right-to-left on the top partition [2^20 - 4 109, 2^20); sparse_call pods whole and on [777, 2^20); the
                SWITCH_CASES, tie_call, only_top_call and top_call as pods; 2^20 nodes (five tree levels) with empty ones
  entry points  isl_place_stream and isl_place_stream_device (batch edges cut would-be runs, later batches free what earlier ones placed),
                isl_place_batch_device and isl_what_if on the top partition of 2^20 GPUs, every policy
"""
import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

from test_oracle_bestfit_limits import HALF, TOP, TOP_LO
from test_oracle_first_available_limits import (BF_POLICIES, EDGE_KINDS, KBF_POLICIES, POLICIES, alt_call, dead15_call, edge_call,
                                                edge_pods, fa_place, fixture_case, good_profiles, podify, top_range)
from test_oracle_gang_topology_limits import FIXTURES
from test_oracle_request_major_limits import eight_gpu_nodes, gang_call, scoring_nodes, top_nodes, whole_bytes
from test_oracle_table_limits import t16x8, t8tab, t8tab_node_tables

pytestmark = pytest.mark.gpu
FA = E.FLAG_FIRST_AVAILABLE
NODE_SCORING = (E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED)
CASES = [("t16x8", E.QUIRKS_REF_EXACT)] + [(f, q) for f in ("t16mix1", "t16mix2") for q in (0, 1, 2, 3)] + [("t8tab", E.QUIRKS_FIXED)]
COUNTERS = ("requests", "placed", "no_capacity", "freed", "batches", "kernel_launches")


class Pair:
    """A flagged engine and one without the flag, same policy, quirks, tables, inventory and partition."""

    def __init__(self, rows, policy, quirks, max_gpus, max_batch=1 << 16):
        self.rows, self.policy, self.quirks = rows, policy, quirks
        self.engs = [E.Engine(max_gpus=max(max_gpus, 4096), max_batch=max_batch, policy=policy, quirks=quirks, flags=f) for f in (FA, 0)]
        for eng in self.engs:
            if rows.ndim == 2:
                eng.load_profile_tables(rows)
            else:
                eng.load_profiles(rows)
        self.eng, self.twin = self.engs

    def load(self, node_off, occ, node_table=None, part=None):
        for eng in self.engs:
            eng.load_inventory(node_off, occ)
            if node_table is not None:
                eng.set_node_tables(node_table)
            if part:
                eng.set_partition(*part)

    def close(self):
        for eng in self.engs:
            eng.close()


def counters(eng):
    s = eng.stats()
    return {k: int(s[k]) for k in COUNTERS}


def check(pair, call, want, want_occ, req, n_names, batches, what, extra=0):
    """Run ``call(engine)`` on both engines; the flagged one's records and occupancy must equal the brute force's, its counters move as
    the records say, and its freed / batches as the unflagged engine's."""
    before = [counters(e) for e in pair.engs]
    got = call(pair.eng)
    call(pair.twin)
    after = [counters(e) for e in pair.engs]
    d = {k: after[0][k] - before[0][k] for k in COUNTERS}
    dt = {k: after[1][k] - before[1][k] for k in COUNTERS}
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(pair.eng.read_occupancy(), want_occ), what
    alloc = req["op"] == E.OP_ALLOC
    placed = int((alloc & (want["status"] == E.ST_PLACED)).sum())
    known = int((alloc & (req["profile"] < n_names)).sum())
    assert (d["requests"], d["placed"], d["no_capacity"]) == (len(req), placed, known - placed), (what, d)
    assert d["kernel_launches"] == 2 * batches + extra, (what, d)
    assert (d["freed"], d["batches"]) == (dt["freed"], dt["batches"]) and d["batches"] == batches, (what, d, dt)
    return got


def batch_case(pair, node_off, occ, req, node_table=None, lo=0, hi=None, how="whole", what=""):
    """One call on a fresh inventory: ``how`` "whole" (isl_place_batch), "range" (isl_place_batch_range(lo, hi)) or "partition"
    (isl_set_partition(lo, hi), then isl_place_batch)."""
    G = int(node_off[-1])
    hi = G if hi is None else hi
    pair.load(node_off, occ, node_table, (lo, hi) if how == "partition" else None)
    want, want_occ, _ = fa_place(node_off, pair.rows, occ, req, pair.policy, pair.quirks, node_table, lo, hi)
    call = (lambda e: e.place_batch_range(lo, hi, req)) if how == "range" else (lambda e: e.place_batch(req))
    return check(pair, call, want, want_occ, req, pair.rows.shape[-1], 1, what)


# ---- every fixture, quirk set and policy -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", CASES, ids=["%s-q%d" % c for c in CASES])
def test_fixtures(name, quirks, policy):
    """k_bestfit: 4 096 and 4 097 GPUs of eight-GPU nodes (one table on both sides of kBfSmemGpus); k_nodefit: 2 048 and 2 049 ragged
    nodes with empty ones (the score trees on both sides of kNfSmemNodes); then a range that cuts nodes at both ends."""
    rows = FIXTURES[name]()
    n_names = rows.shape[-1]
    rng = W.SplitMix64(31000 + 100 * policy + 10 * quirks + len(name))
    pair = Pair(rows, policy, quirks, 1 << 15)
    shapes = [scoring_nodes(rng, n) for n in (2048, 2049)] if policy in NODE_SCORING else [eight_gpu_nodes(G) for G in (4096, 4097)]
    for node_off in shapes:
        G = int(node_off[-1])
        node_table = t8tab_node_tables(rng, len(node_off) - 1) if rows.ndim == 2 else None
        occ = whole_bytes(rng, G)
        batch_case(pair, node_off, occ, alt_call(rng, G, n_names, 1500), node_table, what=G)
    v0, v1 = 3, len(node_off) - 4
    while node_off[v0 + 1] - node_off[v0] < 2:
        v0 += 1
    while node_off[v1 + 1] - node_off[v1] < 2:
        v1 -= 1
    lo, hi = int(node_off[v0]) + 1, int(node_off[v1 + 1]) - 1
    for how in ("range", "partition"):
        batch_case(pair, node_off, occ, alt_call(rng, G, n_names, 1000), node_table, lo, hi, how, (how, lo, hi))
    pair.close()


@pytest.mark.parametrize("policy", BF_POLICIES)
@pytest.mark.parametrize("name", ["t16top", "t16straddle"])
def test_min_frag_scores_above_63(name, policy):
    rows = FIXTURES[name]()
    rng = W.SplitMix64(6300 + policy + len(name))
    pair = Pair(rows, policy, E.QUIRKS_FIXED, 4097)
    for G in (4096, 4097):
        kinds = np.array([0x00, 0x01, 0x81, 0xFF], dtype=np.uint8)
        occ = kinds[(rng.next(G) % np.uint64(4)).astype(np.int64)]
        got = batch_case(pair, eight_gpu_nodes(G), occ, alt_call(rng, G, 16, 1200), what=G)
        assert (got["status"] == E.ST_PLACED).any()
    pair.close()


# ---- block and handle edges, the dead mask ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", [("t16x8", E.QUIRKS_REF_EXACT), ("t8tab", E.QUIRKS_FIXED)])
def test_block_and_handle_edges(name, quirks, policy):
    rng = W.SplitMix64(3232 + policy + len(name))
    rows, node_off, node_table = fixture_case(name, rng, 4096)
    occ = whole_bytes(rng, 4096)
    req, runs, _marks = edge_call(rng, rows.shape[-1], good_profiles(rows, quirks))
    pair = Pair(rows, policy, quirks, 4096)
    got = batch_case(pair, node_off, occ, req, node_table, what="edge call")
    for a, n in runs:
        assert (got["status"][a:a + n] == E.ST_ALT_SKIPPED).sum() > n - 8
    pair.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_profile_15_dead_within_a_launch(policy):
    """Profile 15 dies in batch 1 (first alternative of pods at lanes 0 and 9 of block 0 and at lane 31 of block 2) and places again in
    batch 2 after whole-byte FREEs: two isl_place_batch calls, then the two batches in one isl_place_stream on a fresh inventory."""
    rng = W.SplitMix64(1515 + policy)
    rows, quirks, node_off, occ, b1, b2, full = dead15_call(rng)
    pair = Pair(rows, policy, quirks, 4096)
    pair.load(node_off, occ)
    w1, o1, _ = fa_place(node_off, rows, occ, b1, policy, quirks)
    w2, o2, _ = fa_place(node_off, rows, o1, b2, policy, quirks)
    check(pair, lambda e: e.place_batch(b1), w1, o1, b1, 16, 1, "batch 1")
    got = check(pair, lambda e: e.place_batch(b2), w2, o2, b2, 16, 1, "batch 2")
    assert ((b2["profile"] == 15) & (got["status"] == E.ST_PLACED)).sum() == len(full)
    pair.load(node_off, occ)
    both = np.concatenate([b1, b2])
    check(pair, lambda e: np.concatenate(e.place_stream([b1, b2])), np.concatenate([w1, w2]), o2, both, 16, 2, "stream")
    pair.close()


# ---- 2^20 GPUs ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
def test_2_20_gpus(policy):
    """T8tab with node tables, the lower half and table 7 full: the whole inventory, isl_place_batch_range on the range past the first
    node of table 7 and the same range as a partition; placements above bit 19."""
    rng = W.SplitMix64(TOP + 7 + policy)
    rows, node_off, node_table, occ, req, lo, hi = top_range(rng, n=60 if policy in NODE_SCORING else 150)
    pair = Pair(rows, policy, E.QUIRKS_FIXED, TOP)
    for how in ("whole", "range", "partition"):
        a, b = (0, TOP) if how == "whole" else (lo, hi)
        got = batch_case(pair, node_off, occ, req, node_table, a, b, how, how)
        placed = got[got["status"] == E.ST_PLACED]
        assert ((placed["gpu"] & HALF) != 0).any() and (placed["gpu"] >= a).all()
        p15 = (req["op"] == E.OP_ALLOC) & (req["profile"] == 15) & (got["status"] != E.ST_PLACED)
        assert (got["size"][p15] == rows["size"][7, 15]).all()
    pair.close()


def test_right_to_left_top_partition():
    """T16x8 right-to-left on [2^20 - 4 109, 2^20), which cuts a node: prof.flip under the flag."""
    rng = W.SplitMix64(4109)
    rows = t16x8()
    node_off = eight_gpu_nodes(TOP)
    occ = whole_bytes(rng, TOP, dense=True)
    req = podify(rng, gang_call(rng, TOP, 16, 2000), 16, TOP)
    top = np.flatnonzero(req["op"] == E.OP_FREE)[::2]
    req["handle"][top] = TOP_LO + (req["handle"][top] % np.uint32(TOP - TOP_LO))     # half the FREEs inside the partition
    pair = Pair(rows, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT, TOP)
    got = batch_case(pair, node_off, occ, req, lo=TOP_LO, hi=TOP, how="partition", what="top partition")
    placed = got[got["status"] == E.ST_PLACED]
    assert len(placed) and (placed["gpu"] >= TOP_LO).all() and placed["gpu"].max() >= TOP - 8
    pair.close()


@pytest.mark.parametrize("policy", KBF_POLICIES)
@pytest.mark.parametrize("where", ["whole", "partition"])
def test_sparse_pods(where, policy):
    rng = W.SplitMix64(777 + policy)
    rows, quirks, node_off, node_table, occ, req, lo, hi = edge_pods(rng, "sparse", policy, where)
    pair = Pair(rows, policy, quirks, TOP)
    got = batch_case(pair, node_off, occ, req, lo=lo, hi=hi, how="partition", what=("sparse", where))
    assert (got["status"] == E.ST_PLACED).sum() == 7
    pair.close()


@pytest.mark.parametrize("policy", BF_POLICIES)
@pytest.mark.parametrize("kind", EDGE_KINDS)
def test_edge_pods(kind, policy):
    rng = W.SplitMix64(2020 + len(kind))
    rows, quirks, node_off, node_table, occ, req, lo, hi = edge_pods(rng, kind, policy)
    pair = Pair(rows, policy, quirks, int(node_off[-1]))
    got = batch_case(pair, node_off, occ, req, node_table, lo, hi, "partition", kind)
    assert (got["status"] == E.ST_PLACED).any()
    pair.close()


@pytest.mark.parametrize("policy,name,quirks", [(E.POLICY_MOST_ALLOCATED, "t16x8", E.QUIRKS_REF_EXACT),
                                                (E.POLICY_LEAST_ALLOCATED, "t8tab", E.QUIRKS_FIXED)])
def test_2_20_nodes(policy, name, quirks):
    """2^20 nodes of 0..1 GPUs (five levels of 32-ary score trees in global memory)."""
    rng = W.SplitMix64(1 << 20)
    rows = FIXTURES[name]()
    node_off = top_nodes(rng)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, len(node_off) - 1) if rows.ndim == 2 else None
    occ = whole_bytes(rng, G, dense=True)
    pair = Pair(rows, policy, quirks, TOP)
    got = batch_case(pair, node_off, occ, alt_call(rng, G, 16, 120), node_table, what="2^20 nodes")
    assert (got["status"] == E.ST_PLACED).any()
    pair.close()


# ---- the other entry points on the top partition of 2^20 GPUs -------------------------------------------------------------------------
def top_state(rng, policy):
    """T8tab with node tables on 2^20 GPUs, whole bytes, the partition [2^20 - 4 109, 2^20) loaded on a fresh pair."""
    rows = t8tab()
    node_off = eight_gpu_nodes(TOP)
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    occ = whole_bytes(rng, TOP)
    pair = Pair(rows, policy, E.QUIRKS_FIXED, TOP)
    pair.load(node_off, occ, node_table, (TOP_LO, TOP))
    return pair, rows, node_off, node_table, occ


def frees_of(rng, out):
    """FREEs of about half the PLACED records ``out``."""
    done = out[out["status"] == E.ST_PLACED]
    done = done[rng.next(len(done)) % np.uint64(2) == 0]
    req = np.zeros(len(done), dtype=E.REQUEST_DTYPE)
    req["handle"], req["op"], req["start"], req["size"] = done["gpu"], E.OP_FREE, done["start"], done["size"]
    return req


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_stream(device, policy):
    """Four batches in one isl_place_stream / _device call: each of the three batch edges cuts a run of alternatives in two pods, and each
    later batch frees half of what the batches before it placed (its FREEs sit between two pods in its middle; A2 applies them first)."""
    torch = pytest.importorskip("torch") if device else None
    rng = W.SplitMix64(4444 + policy + 10 * device)
    pair, rows, node_off, node_table, occ = top_state(rng, policy)
    pods = alt_call(rng, TOP, 16, 2400)
    runs = [i for i in range(1, len(pods)) if pods["op"][i] == pods["op"][i - 1] == E.OP_ALLOC and pods["handle"][i] == pods["handle"][i - 1]]
    cuts = [0] + [next(i for i in runs if i >= k) for k in (500, 1100, 1700)] + [len(pods)]
    cur, batches, want, placed = occ, [], [], np.zeros(0, dtype=E.RESULT_DTYPE)
    for b in range(4):
        seg = pods[cuts[b]:cuts[b + 1]]
        mid = next(i for i in range(len(seg) // 2, len(seg)) if seg["op"][i] == E.OP_ALLOC and seg["op"][i - 1] != E.OP_ALLOC)
        req = np.concatenate([seg[:mid], frees_of(rng, placed), seg[mid:]])
        out, cur, _ = fa_place(node_off, rows, cur, req, policy, E.QUIRKS_FIXED, node_table, TOP_LO, TOP)
        batches.append(req)
        want.append(out)
        placed = np.concatenate([placed, out[(req["op"] == E.OP_ALLOC) & (out["status"] == E.ST_PLACED)]])
    req_all, want_all = np.concatenate(batches), np.concatenate(want)
    sizes = np.array([len(b) for b in batches], dtype=np.uint32)

    def call(eng):
        if not device:
            return np.concatenate(eng.place_stream(batches))
        d_in = torch.from_numpy(req_all.view(np.uint8).copy()).cuda()
        d_out = torch.zeros(len(req_all) * 8, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        eng.place_stream_ptr(sizes, d_in.data_ptr(), d_out.data_ptr(), device=True)
        eng.synchronize()
        return d_out.cpu().numpy().view(E.RESULT_DTYPE)
    check(pair, call, want_all, cur, req_all, 16, 4, ("stream", device))
    assert all((b["op"] == E.OP_FREE).any() for b in batches[1:])
    assert all(a["handle"][-1] == b["handle"][0] and a["op"][-1] == b["op"][0] == E.OP_ALLOC for a, b in zip(batches, batches[1:]))
    pair.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_batch_device_and_what_if(policy):
    """isl_place_batch_device, then isl_what_if: its records equal the brute force's, the live state is unchanged, cap_before is
    isl_capacity of the live state and cap_after that of an engine loaded with the brute force's occupancy after the plan."""
    torch = pytest.importorskip("torch")
    rng = W.SplitMix64(5555 + policy)
    pair, rows, node_off, node_table, occ = top_state(rng, policy)
    req = alt_call(rng, TOP, 16, 1500)
    want, cur, _ = fa_place(node_off, rows, occ, req, policy, E.QUIRKS_FIXED, node_table, TOP_LO, TOP)
    d_in = torch.from_numpy(req.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(req) * 8, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def device(eng):
        eng.place_batch_device(len(req), d_in.data_ptr(), d_out.data_ptr())
        eng.synchronize()
        return d_out.cpu().numpy().view(E.RESULT_DTYPE).copy()
    check(pair, device, want, cur, req, 16, 1, "device")
    plan = alt_call(rng, TOP, 16, 1500)
    want, hyp, _ = fa_place(node_off, rows, cur, plan, policy, E.QUIRKS_FIXED, node_table, TOP_LO, TOP)
    live_cap = pair.eng.capacity()
    res = {}

    def what_if(eng):
        out, before, after = eng.what_if(plan)
        if eng is pair.eng:
            res["before"], res["after"] = before, after
        return out
    check(pair, what_if, want, cur, plan, 16, 1, "what_if", extra=2)
    assert np.array_equal(res["before"], live_cap) and np.array_equal(pair.eng.capacity(), live_cap)
    pair.twin.load_inventory(node_off, hyp)
    pair.twin.set_node_tables(node_table)
    pair.twin.set_partition(TOP_LO, TOP)
    assert np.array_equal(res["after"], pair.twin.capacity()) and not np.array_equal(res["after"], live_cap)
    pair.close()
