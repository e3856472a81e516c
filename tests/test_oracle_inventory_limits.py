"""The inventory-size limits of the first-fit paths, and the CPU pins of the oracle there (CPU only).

Three things are sized by the number of GPUs, and ``test_gpu_inventory_limits.py`` runs every one of them at its edge:
  ISL_MAX_GPUS = 2^24   candidate records pack ``gpu << 8 | occ`` into 32 bits; the sweep covers 4 096 GPUs per CTA, 16 per thread
  the full stage        a k_pipeline stage walks up to kSubMax = 8 sub-segments of at most kSegMax = 512 GPUs (max_segment_for)
  the plan arithmetic   which path a call takes: speculative rounds, the plain pipeline, or chunk by chunk (fed host streams keep
                        1 + kFeedReserve SMs free; isl_stream_open plans the same way; the free masks of a stream stay within 256 MiB)

``plan_path`` restates that arithmetic (islplace.cu: route, plan_pipeline, segment_geometry; isl_kernels.cuh: max_segment_for), so
that the GPU tests take every expected path from it with the device's real SM count.  The generators build the occupancies the GPU
tests use, and the self-checks below make sure that, on the oracle, each one reaches the edge it is named for.
"""
import math

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W
from test_oracle_table_limits import candidates, churn_batches

MAX_GPUS = 1 << 24
SWEEP_BLOCK = 4096          # GPUs per sweep CTA (kSweepBlock)
SWEEP_VEC = 16              # GPUs per sweep thread (sweep_mask16)
SEG_MAX, SUB_MAX = 512, 8   # kSegMax, kSubMax
FEED_RESERVE = 3            # kFeedReserve
SPEC_MAX_STAGES = 148       # kSpecMaxStages
CHUNK = 65536               # kChunk: requests per pipeline chunk
MASK_BUDGET = 256 << 20     # bytes of free masks a stream may keep on the device (route)
H100_SMS = 132


# ---- the plan arithmetic, restated -------------------------------------------------------------------------------------------------
def max_segment_for(n_cand):
    """Largest (sub-)segment whose worst-case queue windows fit in the pipeline's shared memory."""
    s = (12288 - (10 + 2 * 32 + 2) * 16) // max(1, n_cand)
    return SEG_MAX if s >= SEG_MAX else s // 64 * 64


def _geometry(G, sms, seg_cap, n_chunks, avg_chunk, fed, spec):
    """segment_geometry: (n_seg, n_sub, sub), or None where it returns ISL_ERANGE.  One pipeline CTA per SM."""
    ceil = lambda a, b: -(-a // b)
    s_opt = math.sqrt(max(1.0, n_chunks - 1.0) * min(avg_chunk, 3.5 * G) * (0.0326 / 1.57))
    target = sms if spec else int(min(sms, max(1.0, math.floor(s_opt + 0.5))))
    reserve = fed and sms > 2 * FEED_RESERVE
    if reserve:
        target = min(target, sms - 1 - FEED_RESERVE)
    if seg_cap < 64:
        return None
    sub = min(seg_cap, max(64, (ceil(G, target) + 63) // 64 * 64))
    stages_avail = sms - 1 - FEED_RESERVE if reserve else sms
    target = max(target, min(stages_avail, ceil(ceil(G, sub), SUB_MAX)))
    n_sub = max(1, ceil(ceil(G, sub), target))
    if n_sub > SUB_MAX:
        return None
    n_seg = max(1, ceil(G, sub * n_sub))
    return None if n_seg > sms else (n_seg, n_sub, sub)


def plan_path(G, sms, n_cand, fed=False, n_batches=1, max_gpus=None, sizes=None, spec=None):
    """Path of an unpartitioned first-fit call of ``n_batches`` mixed batches (``sizes``, default 4 096 requests each) on G GPUs:
    ("spec", 1, sub) for speculative rounds, ("plain", n_sub, sub) for the plain pipeline with n_sub sub-segments per stage, ("chunks",
    None, None) for the chunk-by-chunk path.  ``fed``: a host stream of two or more batches (it keeps 1 + FEED_RESERVE SMs free);
    ``spec``: speculative rounds allowed (default: what ISL_SPEC_AUTO grants, single batches only, without a causal window)."""
    sizes = list(sizes) if sizes is not None else [4096] * n_batches
    assert len(sizes) == n_batches
    max_gpus = G if max_gpus is None else max_gpus
    occ_bytes = -(-max_gpus // SWEEP_BLOCK) * SWEEP_BLOCK
    if n_batches * occ_bytes > MASK_BUDGET:
        return ("chunks", None, None)
    fed = fed and n_batches >= 2
    spec = n_batches == 1 if spec is None else spec
    n_chunks = sum(-(-n // CHUNK) for n in sizes)
    avg = sum(sizes) / n_chunks
    seg_cap = max_segment_for(n_cand)
    if spec:
        g = _geometry(G, sms, seg_cap, n_chunks, avg, fed, True)
        if g is not None and g[1] == 1 and 2 <= g[0] <= SPEC_MAX_STAGES:
            return ("spec", 1, g[2])
    g = _geometry(G, sms, seg_cap, n_chunks, avg, fed, False)
    return ("chunks", None, None) if g is None else ("plain", g[1], g[2])


def stream_open_fits(G, sms, n_cand, max_batches=4):
    """isl_stream_open plans a fed pipeline of max(2, max_batches) full chunks and needs 1 + FEED_RESERVE SMs beside it."""
    g = _geometry(G, sms, max_segment_for(n_cand), max(2, max_batches), CHUNK, True, False)
    return g is not None and g[0] + 1 + FEED_RESERVE <= sms


def full_stage(sms, sub):
    """Every SM's stage holding SUB_MAX sub-segments of ``sub`` GPUs."""
    return sms * SUB_MAX * sub


def fed_reach(sms, sub):
    return (sms - 1 - FEED_RESERVE) * SUB_MAX * sub


def budget_batches(max_gpus):
    """The longest stream whose free masks (one byte per GPU of max_gpus, rounded up to a sweep block, per batch) fit the budget."""
    return MASK_BUDGET // (-(-max_gpus // SWEEP_BLOCK) * SWEEP_BLOCK)


# ---- tables ------------------------------------------------------------------------------------------------------------------------
def k1_rows():
    """The H100 80GB table: 18 candidates under FIXED quirks, 15 under the reference's; k_pipeline<1, ..>, 512-GPU sub-segments."""
    return E.make_profiles(tables.H100_80GB)


def k2_rows():
    """A100 40GB and H100 80GB node tables over one name list: 36 candidates under FIXED quirks (k_pipeline<2, ..>)."""
    return E.make_profile_tables([tables.A100_40GB, tables.H100_80GB])[1]


def k2_node_tables(rng, n_nodes):
    t = (rng.next(n_nodes) & np.uint64(1)).astype(np.uint8)
    t[0] = 1
    return t


def n_names(rows):
    return rows.shape[-1]


# ---- generators ----------------------------------------------------------------------------------------------------------------------
def _partial(rng, n):
    """Occupancy bytes with a few free slices each (never 0xFF, never empty)."""
    b = (rng.next(n) | rng.next(n)) & np.uint64(0xFF)
    b[b == 0xFF] = 0x7F
    b[b == 0] = 0x01
    return b.astype(np.uint8)


def tail_occ(rng, G, sub, n_holes, rtl=False):
    """Full, except ``n_holes`` partly free GPUs spread over the inventory and a partly free last sub-segment of ``sub`` GPUs: the
    stage that holds it is the last one the chain reaches (right-to-left: canonical [0, sub), stored last)."""
    occ = np.full(G, 0xFF, dtype=np.uint8)
    idx = (rng.next(n_holes) % np.uint64(G - sub)).astype(np.int64)
    occ[idx] = _partial(rng, n_holes)
    occ[G - sub:] = _partial(rng, sub)
    return occ[::-1].copy() if rtl else occ


def top_occ(rng, G, n_low=None, block=SWEEP_BLOCK):
    """Mostly full, sparse holes: ``n_low`` partly free GPUs below the last sweep block, 64 in it, a partly free last 16-GPU vector and
    an empty GPU G - 1.  The candidate list stays short and the chain jumps from hole to hole."""
    n_low = max(8, G >> 16) if n_low is None else n_low
    occ = np.full(G, 0xFF, dtype=np.uint8)
    occ[(rng.next(n_low) % np.uint64(G - block)).astype(np.int64)] = _partial(rng, n_low)
    occ[G - block + (rng.next(64) % np.uint64(block - SWEEP_VEC)).astype(np.int64)] = _partial(rng, 64)
    occ[G - SWEEP_VEC:] = _partial(rng, SWEEP_VEC)
    occ[G - 1] = 0
    return occ


def low_half_full(rng, G):
    """The low half full, the high half mostly free: a single profile's capacity sums past 2^24 at this size."""
    occ = np.full(G, 0xFF, dtype=np.uint8)
    occ[G // 2:] = (rng.next(G - G // 2) & rng.next(G - G // 2) & rng.next(G - G // 2) & np.uint64(0xFF)).astype(np.uint8)
    return occ


def top_batches(rng, ref, G, n, frees_top=True):
    """Two mixed batches: the first fills every hole (the last ones at the top), the second FREEs GPU G - 1's placements and re-places
    them, with more FREEs of the first batch's records."""
    req = W.alloc_requests(W.mix_profiles(rng, n))
    res = ref.place(req)
    req2 = W.alloc_requests(W.mix_profiles(rng, n // 4))
    placed = np.flatnonzero(res["status"] == E.ST_PLACED)
    top = [i for i in placed if int(res["gpu"][i]) == G - 1]
    rest = [i for i in placed if int(res["gpu"][i]) != G - 1][: n // 16]
    slots = (rng.next(len(top) + len(rest)) % np.uint64(len(req2))).astype(np.int64)
    for k, i in enumerate(list(top if frees_top else []) + rest):
        req2[slots[k]] = (int(res["gpu"][i]), 0, E.OP_FREE, int(res["start"][i]), int(res["size"][i]))
    return [(req, res), (req2, ref.place(req2))]


def nodes_of(G, per_node=8):
    return W.node_offsets(G // per_node, per_node)


# ---- self-checks: the plan arithmetic at 132 SMs ---------------------------------------------------------------------------------
def test_plan_arithmetic_matches_the_documented_numbers():
    n15, n18 = len(candidates(k1_rows(), E.QUIRKS_REF_EXACT)), len(candidates(k1_rows(), E.QUIRKS_FIXED))
    n36 = len(candidates(k2_rows(), E.QUIRKS_FIXED))
    assert (n15, n18, n36) == (15, 18, 36)
    assert max_segment_for(n18) == 512 and max_segment_for(n15) == 512 and max_segment_for(128) == 64
    assert 33 <= n36 <= 64 and max_segment_for(n36) == 256
    S = H100_SMS
    assert S * SEG_MAX == 67_584 and full_stage(S, 512) == 540_672 and fed_reach(S, 512) == 524_288
    for n in (n15, n18):
        assert plan_path(67_584, S, n) == ("spec", 1, 512)
        assert plan_path(67_584 + 64, S, n)[0] == "plain"
        assert plan_path(540_672, S, n) == ("plain", 8, 512)
        assert plan_path(540_672 + 64, S, n)[0] == "chunks"
    # the fed host stream's reach ends (SMs - 4) x 8 x 512 GPUs; the device stream keeps the pipeline up to the full stage
    assert plan_path(524_288, S, n18, fed=True, n_batches=3) == ("plain", 8, 512)
    assert plan_path(524_288 + 64, S, n18, fed=True, n_batches=3)[0] == "chunks"
    assert plan_path(540_672, S, n18, fed=True, n_batches=3)[0] == "chunks"
    assert plan_path(540_672, S, n18, n_batches=3) == ("plain", 8, 512)
    assert stream_open_fits(524_288, S, n18) and not stream_open_fits(524_288 + 64, S, n18)
    assert not stream_open_fits(540_672 + 64, S, n18) and not stream_open_fits(MAX_GPUS, S, n18)
    # the free-mask budget counts max_gpus, not the loaded G: 496 batches at max_gpus = 540 672, 497 go batch by batch
    assert budget_batches(540_672) == 496
    assert plan_path(4096, S, n18, fed=True, n_batches=496, max_gpus=540_672, sizes=[64] * 496)[0] == "plain"
    assert plan_path(4096, S, n18, fed=True, n_batches=497, max_gpus=540_672, sizes=[64] * 497)[0] == "chunks"
    # K = 2 at its own sub-segment size
    sub = max_segment_for(n36)
    assert plan_path(S * sub, S, n36) == ("spec", 1, sub)
    assert plan_path(S * sub + 64, S, n36)[0] == "plain"
    assert plan_path(full_stage(S, sub), S, n36) == ("plain", 8, sub)
    assert plan_path(full_stage(S, sub) + 64, S, n36)[0] == "chunks"
    # 2^24 GPUs: past every pipeline plan
    assert plan_path(MAX_GPUS, S, n18)[0] == "chunks" and plan_path(MAX_GPUS, S, n18, n_batches=3)[0] == "chunks"


@pytest.mark.parametrize("sms", [78, 114, 132, 148])
def test_plan_boundaries_follow_the_sm_count(sms):
    """The four boundary sizes the GPU file uses land on the four paths for any SM count, the fed reach four stages short."""
    for rows, quirks in ((k1_rows(), E.QUIRKS_FIXED), (k2_rows(), E.QUIRKS_FIXED)):
        n = len(candidates(rows, quirks))
        sub = max_segment_for(n)
        assert plan_path(sms * sub, sms, n)[0] == "spec"
        assert plan_path(sms * sub + 64, sms, n)[0] == "plain"
        assert plan_path(full_stage(sms, sub), sms, n) == ("plain", SUB_MAX, sub)
        assert plan_path(full_stage(sms, sub) + 64, sms, n)[0] == "chunks"
        assert plan_path(fed_reach(sms, sub), sms, n, fed=True, n_batches=3) == ("plain", SUB_MAX, sub)
        assert plan_path(fed_reach(sms, sub) + 64, sms, n, fed=True, n_batches=3)[0] == "chunks"


# ---- self-checks: every generator reaches its edge on the oracle ---------------------------------------------------------------------
def _oracle(G, occ, rows=None, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None, per_node=8):
    rows = k1_rows() if rows is None else rows
    ref = oracle.Fast(nodes_of(G, per_node), rows, quirks, policy=policy, node_table=node_table)
    ref.load(occ)
    return ref


@pytest.mark.parametrize("rtl", [False, True])
def test_top_inventory_reaches_the_last_gpu(rtl):
    """At 2^24 GPUs: a PLACED record on GPU 2^24 - 1, in the last 16-GPU vector and the last sweep block; a FREE naming GPU 2^24 - 1;
    right-to-left, the first placement is GPU 2^24 - 1."""
    G = MAX_GPUS
    rng = W.SplitMix64(24)
    occ = top_occ(rng, G)
    ref = _oracle(G, occ, policy=E.POLICY_RIGHT_TO_LEFT if rtl else E.POLICY_FIRST_FIT)
    (req, res), (req2, res2) = top_batches(rng, ref, G, 6000)
    placed = res["gpu"][res["status"] == E.ST_PLACED].astype(np.int64)
    assert (placed == G - 1).any()
    assert ((placed >= G - SWEEP_VEC) & (placed < G - 1)).any() and ((placed >= G - SWEEP_BLOCK) & (placed < G - SWEEP_VEC)).any()
    assert (placed < G - SWEEP_BLOCK).any()
    if rtl:
        assert int(res["gpu"][np.flatnonzero(res["status"] == E.ST_PLACED)[0]]) == G - 1
    else:
        assert (res["status"] == E.ST_NO_CAPACITY).any()                # every hole filled: the first-fit chain went to the top
    freed = (req2["op"] == E.OP_FREE) & (res2["status"] == E.ST_FREED)
    assert (res2["gpu"][freed] == G - 1).any()
    assert (res2["gpu"][res2["status"] == E.ST_PLACED] == G - 1).any()   # and the freed top GPU is taken again


def test_scan_mode_positions_pass_2_24():
    """A single profile on an inventory whose low half is full: the exclusive scan of capacities passes 2^24 inside the inventory,
    and the batch is placed in the high half from its first GPU on."""
    from range_oracle import capacity_by_hand
    G = MAX_GPUS
    rng = W.SplitMix64(2424)
    occ = low_half_full(rng, G)
    rows = k1_rows()
    cap = capacity_by_hand(rows, E.QUIRKS_REF_EXACT, occ)
    assert int(cap[0]) > (1 << 24)
    ref = _oracle(G, occ)
    req = W.alloc_requests(np.zeros(50_000, dtype=np.uint8))
    res = ref.place(req)
    assert (res["status"] == E.ST_PLACED).all()
    first = int(np.flatnonzero(occ != 0xFF)[0])
    assert first >= G // 2 and int(res["gpu"][0]) == first


@pytest.mark.parametrize("k,rtl", [(1, False), (1, True), (2, False)])
def test_full_stage_tail_receives_placements(k, rtl):
    """At SMs x 8 x sub GPUs the last sub-segment of the last stage (right-to-left: canonical [0, sub)) gets placements, in the mixed
    batch and in every batch of the churn stream."""
    rows = k1_rows() if k == 1 else k2_rows()
    quirks = E.QUIRKS_REF_EXACT if k == 1 else E.QUIRKS_FIXED
    sub = max_segment_for(len(candidates(rows, quirks)))
    G = full_stage(H100_SMS, sub)
    rng = W.SplitMix64(540 + k + rtl)
    occ = tail_occ(rng, G, sub, 4096 // 8, rtl)
    node_table = k2_node_tables(rng, G // 8) if k == 2 else None
    ref = _oracle(G, occ, rows, quirks, E.POLICY_RIGHT_TO_LEFT if rtl else E.POLICY_FIRST_FIT, node_table)
    tail = (lambda g: g < sub) if rtl else (lambda g: g >= G - sub)
    batches = churn_batches(rng, ref, [4096, 4096, 4096], n_names(rows))
    for req, res in batches:
        placed = res["gpu"][(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)].astype(np.int64)
        assert tail(placed).any() and (~tail(placed)).any()


# ---- oracle.Fast against the faithful restatements, on shrunk copies of every generator ---------------------------------------------
def _faithful_agrees(G, occ, batches, rows, quirks, node_table=None, per_node=8):
    fast = oracle.Fast(nodes_of(G, per_node), rows, quirks, node_table=node_table)
    fast.load(occ)
    other = oracle.Faithful(nodes_of(G, per_node), rows, quirks, node_table=node_table)
    other.load_occupancy_as_dangling(occ)
    for i, req in enumerate(batches):
        assert np.array_equal(fast.place(req), other.place(req)), i
        assert np.array_equal(fast.occupancy(), other.occupancy()), i


def _shrunk_batches(rng, occ, G, n_names_, n, rows, quirks, node_table=None, per_node=8):
    ref = oracle.Fast(nodes_of(G, per_node), rows, quirks, node_table=node_table)
    ref.load(occ)
    return [req for req, _ in churn_batches(rng, ref, [n, n, n], n_names_)]


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_fast_vs_faithful_on_shrunk_generators(quirks):
    rng = W.SplitMix64(77 + quirks)
    rows = k1_rows()
    G = 1 << 13
    cases = [top_occ(rng, G, n_low=16, block=1024), low_half_full(rng, G // 4), tail_occ(rng, G // 4, 64, 40)]
    for occ in cases:
        g = len(occ)
        _faithful_agrees(g, occ, _shrunk_batches(rng, occ, g, 6, 300, rows, quirks), rows, quirks)
    # one-GPU nodes (the inventory of 2^24 nodes, shrunk)
    occ = top_occ(rng, 2048, n_low=8, block=512)
    _faithful_agrees(2048, occ, _shrunk_batches(rng, occ, 2048, 6, 200, rows, quirks, per_node=1), rows, quirks, per_node=1)
    # the two-table inventory of the K = 2 cases
    rows2 = k2_rows()
    occ = tail_occ(rng, 2048, 64, 60)
    nt = k2_node_tables(rng, 256)
    _faithful_agrees(2048, occ, _shrunk_batches(rng, occ, 2048, n_names(rows2), 200, rows2, quirks, node_table=nt), rows2, quirks,
                     node_table=nt)


def test_fast_right_to_left_is_first_fit_mirrored():
    """Right-to-left on an occupancy equals first-fit on the mirrored occupancy with the GPU indices mirrored back (uniform nodes)."""
    rng = W.SplitMix64(4321)
    rows = k1_rows()
    G = 4096
    for occ in (top_occ(rng, G, n_low=16, block=1024), tail_occ(rng, G, 64, 50)):
        rtl = _oracle(G, occ, policy=E.POLICY_RIGHT_TO_LEFT)
        ltr = _oracle(G, occ[::-1].copy())
        req = W.alloc_requests(W.mix_profiles(rng, 3000))
        a, b = rtl.place(req), ltr.place(req)
        placed = a["status"] == E.ST_PLACED
        assert np.array_equal(placed, b["status"] == E.ST_PLACED)
        assert np.array_equal(a["gpu"][placed], G - 1 - b["gpu"][placed].astype(np.int64))
        assert np.array_equal(rtl.occupancy(), ltr.occupancy()[::-1])


def test_fast_runs_at_2_24_gpus():
    """Build, load, one batch and the occupancy round trip at ISL_MAX_GPUS, with 2^21 nodes of 8 GPUs and with 2^24 one-GPU nodes."""
    G = MAX_GPUS
    rng = W.SplitMix64(1 << 24)
    occ = top_occ(rng, G)
    for per_node in (8, 1):
        ref = _oracle(G, occ, per_node=per_node)
        assert np.array_equal(ref.occupancy(), occ)
        req = W.alloc_requests(W.mix_profiles(rng, 2000))
        res = ref.place(req)
        after = ref.occupancy()
        placed = res[res["status"] == E.ST_PLACED]
        assert len(placed) and np.array_equal(np.flatnonzero(after != occ), np.unique(placed["gpu"]))
        ref.load(after)
        assert np.array_equal(ref.occupancy(), after)
