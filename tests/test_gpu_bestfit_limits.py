"""k_bestfit at the inventory limits on the H100: isl_place_batch on ISL_POLICY_BEST_FIT / _MIN_FRAG engines and isl_place_gangs on
engines without a gang flag (every policy), on the generators of ``test_oracle_bestfit_limits.py`` (which restates the kernel's
class-minimum walk and shows that each generator reaches its edge).  Every call is compared with ``bestfit_fast`` byte for byte — records,
the whole occupancy and the ``placed`` counter — and its ``kernel_launches`` delta shows the best-fit path ran: k_prepare + k_bestfit,
2 per batch (isl_what_if: 2 more for the two capacities).

  generators    sparse classes and aborted gangs over far minima (batches under best-fit and min-frag, gangs under every policy, whole
                inventories with Gr % 1 024 != 0 and the partition [777, 2^20)); all 2 048 classes live; the shared / global switch of
                the class bitmaps at 4 096 / 4 097 GPUs; ties across 2^19, GPU 2^20 - 1 alone, min-frag scores above 63
  2^20 GPUs     batches under best-fit and min-frag, gangs under every policy; right-to-left gangs also on [2^20 - 4 109, 2^20)
  entry points  isl_place_batch_range, isl_place_stream (later batches free what earlier ones placed), isl_place_batch_device and
                isl_what_if on the top 4 097 GPUs of 2^20
  long batch    more than 65 536 requests on a 4 096-GPU best-fit engine
"""
import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

import bestfit_fast as BF
import range_oracle as RO
from test_oracle_bestfit_limits import (BF_POLICIES, POLICIES, SPARSE_G, SPARSE_LO, SWITCH_CASES, TOP, TOP_LO, abort_call, live_call,
                                        lower_half_full, only_top_call, sparse_call, switch_call, tie_call, top_call)
from test_oracle_gang_topology_limits import small_gangs
from test_oracle_request_major_limits import eight_gpu_nodes, gang_call, gang_offsets, whole_bytes
from test_oracle_table_limits import t16x8

pytestmark = pytest.mark.gpu
WHERE = {"whole": (SPARSE_G, 0, SPARSE_G), "partition": (TOP, SPARSE_LO, TOP)}


def make_engine(rows, policy, quirks, max_gpus=TOP, max_batch=1 << 16):
    eng = E.Engine(max_gpus=max_gpus, max_batch=max_batch, policy=policy, quirks=quirks)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    return eng


def load(eng, node_off, occ, node_table=None, lo=0, hi=None):
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    G = int(node_off[-1])
    if (lo, G if hi is None else hi) != (0, G):
        eng.set_partition(lo, hi)


def placed_of(out, req):
    return int(((out["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)).sum())


def check(eng, call, want, want_occ, req, batches, what, launches_per_batch=2, extra=0):
    """Run ``call``; its records (and the occupancy) must equal the checker's, and the counters show the best-fit path."""
    before = eng.stats()
    got = call()
    after = eng.stats()
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), want_occ), what
    assert after["kernel_launches"] - before["kernel_launches"] == launches_per_batch * batches + extra, (what, after, before)
    assert after["placed"] - before["placed"] == placed_of(want, req), what
    return got


def batch_case(rows, quirks, policy, node_off, occ, req, node_table=None, lo=0, hi=None, what=""):
    G = int(node_off[-1])
    eng = make_engine(rows, policy, quirks, max_gpus=max(G, 4096), max_batch=max(len(req), 4096))
    load(eng, node_off, occ, node_table, lo, hi)
    want, want_occ = BF.place(node_off, rows, occ, req, quirks, policy, node_table, lo, hi)
    got = check(eng, lambda: eng.place_batch(req), want, want_occ, req, 1, what)
    eng.close()
    return got


def gang_case(rows, quirks, policy, node_off, occ, req, off, node_table=None, lo=0, hi=None, what=""):
    G = int(node_off[-1])
    eng = make_engine(rows, policy, quirks, max_gpus=max(G, 4096), max_batch=max(len(req), 4096))
    load(eng, node_off, occ, node_table, lo, hi)
    want, want_occ = BF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
    got = check(eng, lambda: eng.place_gangs(req, off), want, want_occ, req, 1, what)
    eng.close()
    return got


# ---- the generators ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", list(WHERE))
@pytest.mark.parametrize("policy", BF_POLICIES)
def test_sparse_batch(policy, where):
    G, lo, hi = WHERE[where]
    rows, quirks, node_off, occ, req, _off = sparse_call(G, lo, hi, policy)
    got = batch_case(rows, quirks, policy, node_off, occ, req, lo=lo, hi=hi, what=("sparse", where))
    assert (got["status"] == E.ST_PLACED).sum() == 7


@pytest.mark.parametrize("where", list(WHERE))
@pytest.mark.parametrize("policy", POLICIES)
def test_sparse_gangs(policy, where):
    G, lo, hi = WHERE[where]
    rows, quirks, node_off, occ, req, off = sparse_call(G, lo, hi, policy, gangs=True)
    got = gang_case(rows, quirks, policy, node_off, occ, req, off, lo=lo, hi=hi, what=("sparse gangs", where))
    assert got["status"][9] == E.ST_PLACED


@pytest.mark.parametrize("where", list(WHERE))
@pytest.mark.parametrize("policy", POLICIES)
def test_abort_gangs(policy, where):
    G, lo, hi = WHERE[where]
    rows, quirks, node_off, occ, req, off = abort_call(G, lo, hi, policy)
    got = gang_case(rows, quirks, policy, node_off, occ, req, off, lo=lo, hi=hi, what=("abort", where))
    assert (got["status"][4:7] == E.ST_PLACED).all()


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_abort_call_as_a_batch(policy):
    G, lo, hi = WHERE["whole"]
    rows, quirks, node_off, occ, req, _off = abort_call(G, lo, hi, policy)
    got = batch_case(rows, quirks, policy, node_off, occ, req, what="abort as a batch")
    assert (got["status"] == E.ST_PLACED).sum() == 3


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_all_2048_classes_live(policy):
    rng = W.SplitMix64(2048 + policy)
    rows, node_off, node_table, occ, req = live_call(rng, n=3000 if policy == E.POLICY_BEST_FIT else 1000)
    got = batch_case(rows, E.QUIRKS_FIXED, policy, node_off, occ, req, node_table, what="2048 classes")
    assert (got["status"] == E.ST_PLACED).sum() > 100


@pytest.mark.parametrize("policy", BF_POLICIES)
@pytest.mark.parametrize("case", SWITCH_CASES, ids=[c[0] for c in SWITCH_CASES])
def test_shared_global_switch(case, policy):
    rng = W.SplitMix64(4096 + policy + len(case[0]))
    rows, quirks, node_off, node_table, occ, req, lo, hi = switch_call(rng, case, 3000 if policy == E.POLICY_BEST_FIT else 1000)
    got = batch_case(rows, quirks, policy, node_off, occ, req, node_table, lo, hi, what=case[0])
    assert (got["status"] == E.ST_PLACED).any()


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_ties_across_2_19_and_the_last_gpu(policy):
    rows, quirks, node_off, occ, req = tie_call()
    batch_case(rows, quirks, policy, node_off, occ, req, what="ties")
    rows, quirks, node_off, occ, req = only_top_call()
    got = batch_case(rows, quirks, policy, node_off, occ, req, what="last gpu")
    assert got["gpu"][0] == TOP - 1


@pytest.mark.parametrize("name", ["t16top", "t16straddle"])
def test_min_frag_scores_above_63_at_2_20(name):
    rng = W.SplitMix64(63)
    rows, quirks, node_off, occ, req = top_call(rng, name, n=150)
    got = batch_case(rows, quirks, E.POLICY_MIN_FRAG, node_off, occ, req, what=name)
    assert ((req["profile"] == 15) & (got["status"] == E.ST_PLACED)).any()


# ---- 2^20 GPUs ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", BF_POLICIES)
def test_batch_at_2_20_gpus(policy):
    rng = W.SplitMix64(TOP + policy)
    rows, node_off, node_table, occ, req = lower_half_full(rng, n=400)
    got = batch_case(rows, E.QUIRKS_FIXED, policy, node_off, occ, req, node_table, what="2^20 batch")
    assert (got["gpu"][got["status"] == E.ST_PLACED] >= TOP // 2).any()


@pytest.mark.parametrize("policy", POLICIES)
def test_gangs_at_2_20_gpus(policy):
    rng = W.SplitMix64(TOP + 10 + policy)
    rows, node_off, node_table, occ, req = lower_half_full(rng, n=400)
    off = small_gangs(rng, len(req))
    got = gang_case(rows, E.QUIRKS_FIXED, policy, node_off, occ, req, off, node_table, what="2^20 gangs")
    assert (got["status"] == E.ST_GANG_ABORTED).any() and (got["status"] == E.ST_PLACED).any()
    if policy == E.POLICY_RIGHT_TO_LEFT:                # the top partition cuts a node; flip_gpu at the top of the GPU field
        off2 = gang_offsets(rng, "straddle", len(req))
        got = gang_case(rows, E.QUIRKS_FIXED, policy, node_off, occ, req, off2, node_table, TOP_LO, TOP, "top partition")
        assert (got["gpu"][got["status"] == E.ST_PLACED] >= TOP_LO).all() and (got["status"] == E.ST_PLACED).any()


# ---- the other entry points of the best-fit path -----------------------------------------------------------------------------------
def top_state(rng):
    rows = t16x8()
    node_off = eight_gpu_nodes(TOP)
    occ = whole_bytes(rng, TOP, dense=True)
    return rows, node_off, occ, TOP - 4097, TOP


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_batch_range_at_the_top(policy):
    rng = W.SplitMix64(31 + policy)
    rows, node_off, occ, lo, hi = top_state(rng)
    q = E.QUIRKS_REF_EXACT
    eng = make_engine(rows, policy, q)
    load(eng, node_off, occ)
    req = RO.mixed_requests(rng, occ, lo, hi, 16, 3000)
    want, want_occ = BF.place(node_off, rows, occ, req, q, policy, lo=lo, hi=hi)
    got = check(eng, lambda: eng.place_batch_range(lo, hi, req), want, want_occ, req, 1, "range")
    assert (got["status"] == E.ST_PLACED).any() and (got["status"] == E.ST_FREED).any()
    eng.close()


def frees_of(rng, out, share=2):
    """FREE requests of about 1 / share of the PLACED records ``out``."""
    done = out[out["status"] == E.ST_PLACED]
    done = done[rng.next(len(done)) % np.uint64(share) == 0]
    req = np.zeros(len(done), dtype=E.REQUEST_DTYPE)
    req["handle"], req["op"], req["start"], req["size"] = done["gpu"], E.OP_FREE, done["start"], done["size"]
    return req


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_stream_at_the_top(policy):
    """Four batches in one isl_place_stream call on the partition [2^20 - 4 097, 2^20): each later batch frees half of what the batches
    before it placed, then allocates again."""
    rng = W.SplitMix64(37 + policy)
    rows, node_off, occ, lo, hi = top_state(rng)
    q = E.QUIRKS_REF_EXACT
    eng = make_engine(rows, policy, q)
    load(eng, node_off, occ, lo=lo, hi=hi)
    cur = occ
    batches, want, placed = [], [], np.zeros(0, dtype=E.RESULT_DTYPE)
    for b in range(4):
        allocs = W.alloc_requests((rng.next(900) % np.uint64(16)).astype(np.uint8))
        req = np.concatenate([frees_of(rng, placed), allocs])
        req = req[rng.next(len(req)).argsort()]
        out, cur = BF.place(node_off, rows, cur, req, q, policy, lo=lo, hi=hi)
        batches.append(req)
        want.append(out)
        placed = np.concatenate([placed, out[(req["op"] == E.OP_ALLOC) & (out["status"] == E.ST_PLACED)]])
    assert all((r["op"] == E.OP_FREE).any() for r in batches[1:])
    req_all, want_all = np.concatenate(batches), np.concatenate(want)
    check(eng, lambda: np.concatenate(eng.place_stream(batches)), want_all, cur, req_all, 4, "stream")
    eng.close()


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_batch_device_at_2_20(policy):
    import torch
    rng = W.SplitMix64(41 + policy)
    rows, node_off, occ, _lo, _hi = top_state(rng)
    q = E.QUIRKS_REF_EXACT
    eng = make_engine(rows, policy, q)
    load(eng, node_off, occ)
    req = gang_call(rng, TOP, 16, 400)
    want, want_occ = BF.place(node_off, rows, occ, req, q, policy)
    d_in = torch.from_numpy(req.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(req) * 8, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def call():
        eng.place_batch_device(len(req), d_in.data_ptr(), d_out.data_ptr())
        eng.synchronize()
        return d_out.cpu().numpy().view(E.RESULT_DTYPE)
    check(eng, call, want, want_occ, req, 1, "device")
    eng.close()


@pytest.mark.parametrize("policy", BF_POLICIES)
def test_what_if_at_the_top(policy):
    """isl_what_if on the partition [2^20 - 4 097, 2^20): the plan's records as the checker's, capacity before and after as counted by
    hand on the partition, and the live occupancy back afterwards."""
    rng = W.SplitMix64(43 + policy)
    rows, node_off, occ, lo, hi = top_state(rng)
    q = E.QUIRKS_REF_EXACT
    eng = make_engine(rows, policy, q)
    load(eng, node_off, occ, lo=lo, hi=hi)
    plan = RO.mixed_requests(rng, occ, lo, hi, 16, 2000)
    want, hyp = BF.place(node_off, rows, occ, plan, q, policy, lo=lo, hi=hi)
    res = {}

    def call():
        res["out"], res["before"], res["after"] = eng.what_if(plan)
        return res["out"]
    check(eng, call, want, occ, plan, 1, "what_if", extra=2)
    assert np.array_equal(res["before"], RO.capacity_by_hand(rows, q, occ[lo:hi]))
    assert np.array_equal(res["after"], RO.capacity_by_hand(rows, q, hyp[lo:hi]))
    assert not np.array_equal(res["before"], res["after"])
    eng.close()


def test_more_than_65536_requests_on_4096_gpus():
    rng = W.SplitMix64(65537)
    rows = t16x8()
    G = 4096
    node_off = eight_gpu_nodes(G)
    occ = whole_bytes(rng, G)
    req = gang_call(rng, G, 16, 70000)
    req["op"][(rng.next(len(req)) % np.uint64(8) != 0) & (req["op"] == E.OP_ALLOC)] = E.OP_NOOP     # room lasts past request 65 536
    got = batch_case(rows, E.QUIRKS_REF_EXACT, E.POLICY_BEST_FIT, node_off, occ, req, what="70 000 requests")
    assert (got["status"][65536:] == E.ST_PLACED).sum() > 100
