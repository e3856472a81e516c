"""The first-fit paths at the inventory limits (the fixtures, the plan restatement and their self-checks are in
``test_oracle_inventory_limits.py``).  Every call is compared with ``oracle.Fast`` byte for byte — records and final occupancy — and
every case about a path proves which path ran through the engine's ``kernel_launches`` / ``spec_chunks`` counters:
  speculative rounds   3 launches (k_prepare, k_partition, k_pipeline), one speculative cell per chunk
  plain pipeline       3 launches, or 3 per batch + 1 for a fed host stream (copy + pre-pass + ready flag per batch on the feed stream)
  chunk by chunk       per batch k_prepare, per chunk k_partition, two sweeps, k_chain, k_commit
The expected path comes from ``plan_path`` with the device's SM count.  Needs an H100.
"""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W
from range_oracle import RangeFast, capacity_by_hand
from test_oracle_inventory_limits import (CHUNK, MAX_GPUS, SWEEP_BLOCK, SWEEP_VEC, budget_batches, fed_reach, full_stage, k1_rows,
                                          k2_node_tables, k2_rows, low_half_full, max_segment_for, n_names, nodes_of, plan_path,
                                          stream_open_fits, tail_occ, top_batches, top_occ)
from test_oracle_table_limits import candidates, churn_batches

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def make_engine(rows, G, occ, quirks, node_table=None, policy=E.POLICY_FIRST_FIT, max_gpus=None, max_batch=1 << 17, per_node=8):
    eng = E.Engine(max_gpus=max_gpus or max(4096, G), max_batch=max_batch, quirks=quirks, policy=policy)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    eng.load_inventory(nodes_of(G, per_node), occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def make_oracle(rows, G, occ, quirks, node_table=None, policy=E.POLICY_FIRST_FIT, per_node=8):
    ref = oracle.Fast(nodes_of(G, per_node), rows, quirks, policy=policy, node_table=node_table)
    ref.load(occ)
    return ref


def delta(eng, before):
    after = eng.stats()
    return {k: after[k] - before[k] for k in ("kernel_launches", "spec_chunks", "scan_placed", "placed")}


def same(got, want, what):
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])


def expect_path(d, path, sizes, fed=False):
    """The counters of one call that took ``path`` over batches of ``sizes`` requests."""
    chunks = sum(-(-n // CHUNK) for n in sizes)
    if path == "chunks":
        assert d["kernel_launches"] == sum(1 + 5 * -(-n // CHUNK) for n in sizes) and d["spec_chunks"] == 0, (path, d)
    else:
        assert d["kernel_launches"] == (3 * len(sizes) + 1 if fed else 3), (path, fed, d)
        assert d["spec_chunks"] == (chunks if path == "spec" else 0), (path, d)


def device_stream(eng, batches):
    """place_stream_device of the batches; returns the records per batch."""
    import torch
    sizes = np.array([len(r) for r, _ in batches], dtype=np.uint32)
    d_in = torch.from_numpy(np.concatenate([r for r, _ in batches]).view(np.int64).copy()).cuda()
    d_out = torch.zeros_like(d_in)
    torch.cuda.synchronize()
    eng.place_stream_ptr(sizes, d_in.data_ptr(), d_out.data_ptr(), device=True)
    eng.synchronize()
    return np.split(d_out.cpu().numpy().view(E.RESULT_DTYPE), np.cumsum(sizes)[:-1])


def run_three_ways(rows, G, occ, quirks, sms, sub, node_table=None, policy=E.POLICY_FIRST_FIT, seed=0, n=4096):
    """One mixed batch, then a three-batch churn stream with FREEs through place_stream (fed) and place_stream_device, each on a fresh
    inventory; every path asserted from the plan restatement.  The last sub-segment of the last stage receives placements."""
    rtl = policy == E.POLICY_RIGHT_TO_LEFT
    n_cand = len(candidates(rows, quirks))
    tail = (lambda g: g < sub) if rtl else (lambda g: g >= G - sub)
    rng = W.SplitMix64(seed)
    eng = make_engine(rows, G, occ, quirks, node_table, policy)
    # one mixed host batch
    ref = make_oracle(rows, G, occ, quirks, node_table, policy)
    (req, want), = churn_batches(rng, ref, [n], n_names(rows))
    assert tail(want["gpu"][want["status"] == E.ST_PLACED].astype(np.int64)).any()
    before = eng.stats()
    same(eng.place_batch(req), want, (G, "batch"))
    assert np.array_equal(eng.read_occupancy(), ref.occupancy()), (G, "batch")
    path = plan_path(G, sms, n_cand, sizes=[n])[0]
    expect_path(delta(eng, before), path, [n])
    paths = [path]
    # a churn stream, host (fed) and device
    for fed in (True, False):
        eng.load_inventory(nodes_of(G), occ)
        if node_table is not None:
            eng.set_node_tables(node_table)
        ref = make_oracle(rows, G, occ, quirks, node_table, policy)
        batches = churn_batches(rng, ref, [n, n + 1000, n + 2000], n_names(rows))
        for r, w in batches:
            assert tail(w["gpu"][(r["op"] == E.OP_ALLOC) & (w["status"] == E.ST_PLACED)].astype(np.int64)).any()
        before = eng.stats()
        got = eng.place_stream([r for r, _ in batches]) if fed else device_stream(eng, batches)
        for i, (g, (_, w)) in enumerate(zip(got, batches)):
            same(g, w, (G, fed, i))
        assert np.array_equal(eng.read_occupancy(), ref.occupancy()), (G, fed)
        sizes = [len(r) for r, _ in batches]
        path = plan_path(G, sms, n_cand, fed=fed, n_batches=3, sizes=sizes)[0]
        expect_path(delta(eng, before), path, sizes, fed=fed and path != "chunks")
        paths.append(path)
    eng.close()
    return paths


# ---- 1. pipeline boundaries for K = 1 and K = 2 ------------------------------------------------------------------------------------
BOUNDARIES = ["spec", "spec+64", "full", "full+64"]


def boundary_G(which, sms, sub):
    return {"spec": sms * sub, "spec+64": sms * sub + 64, "full": full_stage(sms, sub), "full+64": full_stage(sms, sub) + 64}[which]


@pytest.mark.parametrize("which", BOUNDARIES)
@pytest.mark.parametrize("k", [1, 2])
def test_pipeline_boundaries(k, which, sms):
    """K = 1: the H100 table (15 candidates, 512-GPU sub-segments); K = 2: A100 + H100 node tables (36 candidates, 256-GPU
    sub-segments).  At SMs x sub a batch takes speculative rounds, 64 GPUs more the plain pipeline, at SMs x 8 x sub every stage is
    full, 64 GPUs more the chunk path.  The fed host stream at the full stage is already past its reach."""
    rows = k1_rows() if k == 1 else k2_rows()
    quirks = E.QUIRKS_REF_EXACT if k == 1 else E.QUIRKS_FIXED
    sub = max_segment_for(len(candidates(rows, quirks)))
    assert sub == (512 if k == 1 else 256)
    G = boundary_G(which, sms, sub)
    rng = W.SplitMix64(1000 * k + G)
    node_table = k2_node_tables(rng, G // 8) if k == 2 else None
    occ = tail_occ(rng, G, sub, 4096 // 8)
    paths = run_three_ways(rows, G, occ, quirks, sms, sub, node_table, seed=G + k)
    want = {"spec": ["spec", "plain", "plain"], "spec+64": ["plain", "plain", "plain"], "full": ["plain", "chunks", "plain"],
            "full+64": ["chunks", "chunks", "chunks"]}[which]
    assert paths == want, paths


@pytest.mark.parametrize("variant", ["right_to_left", "fixed"])
def test_full_stage_variants(variant, sms):
    """The full stage (SMs x 8 x 512 GPUs) under ISL_POLICY_RIGHT_TO_LEFT (canonical [0, 512) is the last sub-segment of the last stage
    in storage order) and under ISL_QUIRKS_FIXED (18 candidates, still 512-GPU sub-segments)."""
    rows = k1_rows()
    quirks = E.QUIRKS_FIXED if variant == "fixed" else E.QUIRKS_REF_EXACT
    policy = E.POLICY_RIGHT_TO_LEFT if variant == "right_to_left" else E.POLICY_FIRST_FIT
    sub = max_segment_for(len(candidates(rows, quirks)))
    G = full_stage(sms, sub)
    rng = W.SplitMix64(7000 + len(variant))
    occ = tail_occ(rng, G, sub, 4096 // 8, rtl=policy == E.POLICY_RIGHT_TO_LEFT)
    assert run_three_ways(rows, G, occ, quirks, sms, sub, policy=policy, seed=G + len(variant)) == ["plain", "chunks", "plain"]


# ---- 2. the fed-stream and open-stream reach --------------------------------------------------------------------------------------
def open_stream_batches(eng, ref, rng, n_batches, n):
    """Strictly causal batches through an open stream with pinned buffers: batch b FREEs placements of earlier batches."""
    h_in = E.PinnedArray(n_batches * n, E.REQUEST_DTYPE)
    h_out = E.PinnedArray(n_batches * n, E.RESULT_DTYPE)
    eng.stream_open(n_batches)
    live = []
    for b in range(n_batches):
        req = W.alloc_requests(W.mix_profiles(rng, n))
        for _ in range(min(len(live), n // 3)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        h_in.array[b * n:(b + 1) * n] = req
        t = eng.stream_submit_ptr(n, h_in.ptr + 8 * b * n, h_out.ptr + 8 * b * n)
        eng.stream_wait(t)
        got = h_out.array[b * n:(b + 1) * n].copy()
        same(got, ref.place(req), ("open", b))
        live.extend((int(r["gpu"]), int(r["start"]), int(r["size"])) for r in got[(req["op"] == E.OP_ALLOC) & (got["status"] == E.ST_PLACED)])
    eng.stream_close()
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    h_in.free(); h_out.free()


def erange(fn, *args):
    with pytest.raises(E.EngineError) as ei:
        fn(*args)
    assert ei.value.code == E.ERANGE, ei.value.code


@pytest.mark.parametrize("beyond", [False, True])
def test_fed_and_open_stream_reach(beyond, sms):
    """(SMs - 4) x 8 x 512 GPUs: the fed host stream and isl_stream_open still fit beside the feed reserve; 64 GPUs more the host stream
    takes the chunk path and isl_stream_open returns ISL_ERANGE, while the device stream stays on the pipeline at both sizes.  After the
    refusal the engine is not in the open-stream state."""
    rows, quirks = k1_rows(), E.QUIRKS_REF_EXACT
    n_cand = len(candidates(rows, quirks))
    G = fed_reach(sms, 512) + (64 if beyond else 0)
    rng = W.SplitMix64(5000 + beyond)
    occ = tail_occ(rng, G, 512, 4096 // 8)
    paths = run_three_ways(rows, G, occ, quirks, sms, 512, seed=G)
    assert paths[1:] == (["chunks", "plain"] if beyond else ["plain", "plain"]), paths
    assert stream_open_fits(G, sms, n_cand) == (not beyond)
    n_batches = 3
    eng = make_engine(rows, G, occ, quirks, max_batch=n_batches * CHUNK)
    ref = make_oracle(rows, G, occ, quirks)
    if beyond:
        erange(eng.stream_open, n_batches)
        req = W.alloc_requests(W.mix_profiles(rng, 5000))
        same(eng.place_batch(req), ref.place(req), "after the refusal")
        assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    else:
        open_stream_batches(eng, ref, rng, n_batches, 4096)
    eng.close()


# ---- 3. ISL_MAX_GPUS -----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def top_inventory():
    rng = W.SplitMix64(1 << 24)
    return top_occ(rng, MAX_GPUS)


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_placement_at_2_24_gpus(policy, top_inventory, sms):
    """2^21 nodes of 8 GPUs, mostly full with sparse holes up to GPU 2^24 - 1: a mixed batch on the chunk path, a batch that FREEs the
    top GPU's placements, isl_free_batch of the top GPU, a batch of <= 1 024 requests (k_small's range ends at 2^18: chunk path),
    place_batch_range over the last 16 GPUs and a partition over the top 4 096 + 13 GPUs.  Right-to-left stores canonical GPU 2^24 - 1
    at index 0."""
    G, rows, quirks = MAX_GPUS, k1_rows(), E.QUIRKS_REF_EXACT
    occ = top_inventory
    rng = W.SplitMix64(240 + policy)
    eng = make_engine(rows, G, occ, quirks, policy=policy)
    ref = make_oracle(rows, G, occ, quirks, policy=policy)
    batches = top_batches(rng, ref, G, 6000)
    for i, (req, want) in enumerate(batches):
        before = eng.stats()
        same(eng.place_batch(req), want, ("top", i))
        assert plan_path(G, sms, len(candidates(rows, quirks)), sizes=[len(req)])[0] == "chunks"
        expect_path(delta(eng, before), "chunks", [len(req)])
    assert (batches[0][1]["gpu"] == G - 1).any() and (batches[1][1]["gpu"][batches[1][0]["op"] == E.OP_FREE] == G - 1).any()
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    # isl_free_batch of everything on the top GPU, then a small batch over the whole range
    live = ref.occupancy()
    spans = np.zeros(1, dtype=E.SPAN_DTYPE)
    spans[0] = (G - 1, 0, 8, 0)
    eng.free_batch(spans)
    live[G - 1] = 0
    assert np.array_equal(eng.read_occupancy()[G - SWEEP_BLOCK:], live[G - SWEEP_BLOCK:])
    ref = make_oracle(rows, G, live, quirks, policy=policy)
    small = W.alloc_requests(W.mix_profiles(rng, 1000))
    before = eng.stats()
    want = ref.place(small)
    same(eng.place_batch(small), want, "small")
    expect_path(delta(eng, before), "chunks", [len(small)])
    assert (want["gpu"] == G - 1).any() or policy == E.POLICY_FIRST_FIT
    live = ref.occupancy()
    assert np.array_equal(eng.read_occupancy(), live)
    # the last 16 GPUs through place_batch_range: k_few (<= 8 inline requests) and k_small
    for n in (8, 40):
        req = W.alloc_requests(W.mix_profiles(rng, n))
        rref = RangeFast(nodes_of(G), rows, live, G - SWEEP_VEC, G, quirks, policy)
        same(eng.place_batch_range(G - SWEEP_VEC, G, req), rref.place(req), ("range", n))
        live = rref.occupancy()
        assert np.array_equal(eng.read_occupancy()[G - SWEEP_BLOCK:], live[G - SWEEP_BLOCK:])
    # a partition over the top 4 096 + 13 GPUs (the last sweep block and 13 GPUs of the one before)
    lo = G - SWEEP_BLOCK - 13
    occ2 = live.copy()
    occ2[lo:] = (rng.next(G - lo) & rng.next(G - lo) & np.uint64(0xFF)).astype(np.uint8)
    eng.write_occupancy(lo, occ2[lo:])
    eng.set_partition(lo, G)
    req = W.alloc_requests(W.mix_profiles(rng, 3000))
    rref = RangeFast(nodes_of(G), rows, occ2, lo, G, quirks, policy)
    same(eng.place_batch(req), rref.place(req), "partition")
    assert np.array_equal(eng.read_occupancy(), rref.occupancy())
    eng.close()


def test_scan_mode_at_2_24_gpus(sms):
    """A single profile on 2^24 GPUs whose low half is full: the chunk path's scan mode, capacity positions past 2^24."""
    G, rows, quirks = MAX_GPUS, k1_rows(), E.QUIRKS_REF_EXACT
    rng = W.SplitMix64(2424)
    occ = low_half_full(rng, G)
    assert int(capacity_by_hand(rows, quirks, occ)[0]) > (1 << 24)
    eng = make_engine(rows, G, occ, quirks)
    ref = make_oracle(rows, G, occ, quirks)
    req = W.alloc_requests(np.zeros(50_000, dtype=np.uint8))
    before = eng.stats()
    same(eng.place_batch(req), ref.place(req), "scan")
    d = delta(eng, before)
    assert d["scan_placed"] == d["placed"] == 50_000, d
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    eng.close()


def test_queries_at_2_24_gpus(top_inventory):
    """isl_capacity, isl_what_if, snapshot / restore, isl_write_occupancy of the last byte, isl_gpu_to_node of the last GPU (also with
    2^24 one-GPU nodes), and a load of 2^24 + 1 GPUs refused with the previous inventory kept."""
    G, rows, quirks = MAX_GPUS, k1_rows(), E.QUIRKS_REF_EXACT
    occ = top_inventory
    rng = W.SplitMix64(99)
    eng = make_engine(rows, G, occ, quirks)
    assert np.array_equal(eng.capacity(), capacity_by_hand(rows, quirks, occ))
    ref = make_oracle(rows, G, occ, quirks)
    plan = W.alloc_requests(W.mix_profiles(rng, 3000))
    plan[0] = (G - 1, 0, E.OP_FREE, 0, 1)
    busy = np.flatnonzero(occ[: G - 1] == 0xFF)[-5:]
    for i, g in enumerate(busy):
        plan[1 + i] = (int(g), 0, E.OP_FREE, 0, 2)
    got, cap_before, cap_after = eng.what_if(plan)
    same(got, ref.place(plan), "what_if")
    assert np.array_equal(cap_before, capacity_by_hand(rows, quirks, occ))
    assert np.array_equal(cap_after, capacity_by_hand(rows, quirks, ref.occupancy()))
    assert np.array_equal(eng.read_occupancy(), occ)
    # snapshot, place, restore
    eng.snapshot_occupancy()
    ref = make_oracle(rows, G, occ, quirks)
    req = W.alloc_requests(W.mix_profiles(rng, 5000))
    same(eng.place_batch(req), ref.place(req), "before restore")
    assert eng.read_occupancy()[G - 1] != 0
    eng.restore_occupancy()
    assert np.array_equal(eng.read_occupancy(), occ)
    # the last byte, and one past it
    eng.write_occupancy(G - 1, np.array([0x0F], dtype=np.uint8))
    live = occ.copy()
    live[G - 1] = 0x0F
    assert np.array_equal(eng.read_occupancy(), live)
    erange(eng.write_occupancy, G - 1, np.zeros(2, dtype=np.uint8))
    assert np.array_equal(eng.read_occupancy(), live)
    assert eng.gpu_to_node(G - 1) == (G >> 3) - 1 and eng.gpu_to_node(G) == E.GPU_NONE
    # one GPU too many: refused, the inventory stays
    big = np.concatenate([nodes_of(G), [G + 1]]).astype(np.uint32)
    erange(eng.load_inventory, big, np.zeros(G + 1, dtype=np.uint8))
    assert eng.num_gpus == G and np.array_equal(eng.read_occupancy(), live)
    ref = make_oracle(rows, G, live, quirks)
    req = W.alloc_requests(W.mix_profiles(rng, 2000))
    same(eng.place_batch(req), ref.place(req), "after the refused load")
    # 2^24 one-GPU nodes
    eng.load_inventory(nodes_of(G, 1), occ)
    assert eng.gpu_to_node(G - 1) == G - 1 and eng.gpu_to_node(0) == 0
    ref = make_oracle(rows, G, occ, quirks, per_node=1)
    req = W.alloc_requests(W.mix_profiles(rng, 6000))
    same(eng.place_batch(req), ref.place(req), "one-GPU nodes")
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    # an open stream cannot plan 2^24 GPUs, and the engine stays usable
    erange(eng.stream_open, 2)
    req = W.alloc_requests(W.mix_profiles(rng, 2000))
    same(eng.place_batch(req), ref.place(req), "after the refused open stream")
    eng.close()


def test_partitioned_halves_at_2_24_gpus(top_inventory):
    """isl_place_batch_partitioned with two engines of 2^23 GPUs each, the queue-head token carried by the caller; the minimum of the
    two result arrays is the global first-fit."""
    import torch
    G, rows, quirks = MAX_GPUS, k1_rows(), E.QUIRKS_REF_EXACT
    occ = top_inventory
    rng = W.SplitMix64(23)
    ref = make_oracle(rows, G, occ, quirks)
    req = W.alloc_requests(W.mix_profiles(rng, 6000))
    want = ref.place(req)
    assert (want["gpu"] == G - 1).any() and (want["gpu"][want["status"] == E.ST_PLACED] < G // 2).any()
    d_in = torch.from_numpy(req.view(np.int64).copy()).cuda()
    heads = torch.zeros(2 * 16, dtype=torch.int32, device="cuda")
    outs, engines = [], []
    for r, (lo, hi) in enumerate(((0, G // 2), (G // 2, G))):
        eng = make_engine(rows, G, occ, quirks)
        eng.set_partition(lo, hi)
        out = torch.empty_like(d_in)
        nxt = torch.zeros_like(heads)
        torch.cuda.synchronize()
        eng.place_batch_partitioned(len(req), d_in.data_ptr(), out.data_ptr(), heads.data_ptr() if r else None, nxt.data_ptr())
        eng.synchronize()
        heads = nxt
        outs.append(out.cpu().numpy())
        engines.append((eng, lo, hi))
    same(np.minimum(outs[0], outs[1]).view(E.RESULT_DTYPE), want, "partitioned")
    got = np.concatenate([eng.read_occupancy()[lo:hi] for eng, lo, hi in engines])
    assert np.array_equal(got, ref.occupancy())
    for eng, _, _ in engines:
        eng.close()


# ---- 4. the free-mask budget --------------------------------------------------------------------------------------------------------
def test_free_mask_budget(sms):
    """max_gpus = SMs x 8 x 512 with 4 096 GPUs loaded: the budget counts max_gpus.  A host stream of floor(256 MiB / occ_bytes) small
    batches runs as one fed pipeline launch, one batch more runs batch by batch; both bit-exact, FREEs of earlier batches throughout."""
    rows, quirks = k1_rows(), E.QUIRKS_REF_EXACT
    n_cand = len(candidates(rows, quirks))
    max_gpus, G, n = full_stage(sms, 512), 4096, 64
    nb = budget_batches(max_gpus)
    rng = W.SplitMix64(256)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    eng = make_engine(rows, G, occ, quirks, max_gpus=max_gpus, max_batch=(nb + 1) * n)
    for count, path in ((nb, "plain"), (nb + 1, "chunks")):
        assert plan_path(G, sms, n_cand, fed=True, n_batches=count, max_gpus=max_gpus, sizes=[n] * count)[0] == path
        eng.load_inventory(nodes_of(G), occ)
        ref = make_oracle(rows, G, occ, quirks)
        batches = churn_batches(rng, ref, [n] * count, n_names(rows))
        before = eng.stats()
        got = eng.place_stream([r for r, _ in batches])
        for i, (g, (_, w)) in enumerate(zip(got, batches)):
            same(g, w, (count, i))
        assert np.array_equal(eng.read_occupancy(), ref.occupancy()), count
        expect_path(delta(eng, before), path, [n] * count, fed=True)
    eng.close()
