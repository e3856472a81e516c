"""Every placement path on restricted GPU ranges that start and end anywhere: isl_place_batch_range (one node's GPUs, the reference's
findDeviceForASlice), isl_set_partition on a single engine, and ISL_FLAG_ALL_NODES (one restricted pass per node).  Each call is compared
byte for byte with the CPU restatement of ``range_oracle.py`` — records and the WHOLE occupancy, so the bytes outside the range are
checked too — and the engine's counters show that the intended path ran.  Needs an H100.

Path fingerprints (kernel launches per call): k_few / k_small 1; the chunk path 1 + 5 per 65 536-request chunk (1 + 3 on an empty range,
which has no sweep); k_pipeline 3 (k_prepare, k_partition, the pipeline); k_bestfit 2.  A cooperative launch the shared GPU refuses falls
back to the chunk path: the path assertion is then replaced by a warning, the parity assertion stays.
"""
import os
import warnings

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W

import gang_oracle as GO
from range_oracle import RangeFast, capacity_by_hand, mixed_requests, place_range

pytestmark = pytest.mark.gpu
MIX_NAMES = [tables.A100_40GB, tables.H100_80GB, tables.A30_24GB]
SMALL_LIMIT = 1 << 18           # k_small's range limit
FEW_GPUS = 16384                # k_few's: hi - (lo & ~15)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tables_for(n_tables, n_nodes, rng):
    if n_tables == 1:
        rows = E.make_profiles(tables.H100_80GB)
        return rows, None, len(rows)
    names, rows = E.make_profile_tables(MIX_NAMES)
    return rows, (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8), len(names)


def make_engine(node_off, rows, occ, policy, quirks, node_table=None, flags=0, max_batch=1 << 17):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if rows.ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    load(eng, node_off, occ, node_table)
    return eng


def load(eng, node_off, occ, node_table):
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)


def random_occ(rng, G):
    return ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)


def delta(eng, before):
    after = eng.stats()
    return {k: after[k] - before[k] for k in ("kernel_launches", "spec_chunks", "scan_placed", "placed")}


def spec_expected(G, lo, hi, n_tables):
    """Speculative rounds for one mixed batch: one sub-segment per stage (G <= SMs x 512 with the one-table candidate count) and at least
    two stages over the range.  Conservative: only the geometries the plan certainly gives."""
    if n_tables != 1:
        return False
    sms = sm_count()
    sub = min(512, max(64, (-(-G // sms) + 63) // 64 * 64))
    if -(-G // sub) > sms:
        return False
    return -(-(hi - lo) // sub) >= 2


def check_path(d, path, n, what, G=0, lo=0, hi=0, n_tables=1):
    """``path``: "one" (k_few / k_small), "chunks", "scan", "pipeline", "spec" (pipeline with speculative rounds expected when the
    geometry gives them), "plain" (pipeline, speculation off), "bestfit"."""
    chunks = -(-n // 65536)
    empty = hi == lo
    if path in ("pipeline", "spec", "plain") and not empty:
        if d["kernel_launches"] == 2 + 1 + 5 * chunks and d["spec_chunks"] == 0:
            warnings.warn(f"{what}: the cooperative pipeline launch was refused (shared GPU); the chunk path ran, path not checked")
            return
        assert d["kernel_launches"] == 3, (what, d)
        if path == "plain":
            assert d["spec_chunks"] == 0, (what, d)
        elif path == "spec" and spec_expected(G, lo, hi, n_tables):
            assert d["spec_chunks"] == chunks, (what, d)
        return
    if path == "bestfit":
        assert d["kernel_launches"] == (1 if empty else 2), (what, d)
        return
    if path == "one" and not empty and hi - lo <= SMALL_LIMIT:
        assert d["kernel_launches"] == 1, (what, d)
        return
    assert d["kernel_launches"] == (1 + 3 * chunks if empty else 1 + 5 * chunks), (what, path, d)      # the chunk path
    assert d["spec_chunks"] == 0, (what, d)
    if path == "scan":
        assert d["scan_placed"] == d["placed"], (what, d)


def compare(got, want, occ_got, occ_want, what):
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    diff = np.flatnonzero(occ_got != occ_want)
    assert len(diff) == 0, (what, "occupancy", diff[:5], occ_got[diff[:5]], occ_want[diff[:5]])


# ---- (a) isl_place_batch_range: every path, ranges that start and end anywhere ---------------------------------------------------------
def range_bounds(G):
    b = [(0, G), (1, G - 1), (3, 19), (15, 17), (8 * 5, 8 * 6), (511, 513), (513, 4099), (4095, 8193), (16, 16 + FEW_GPUS),
         (8, 8 + FEW_GPUS), (1, 1 + SMALL_LIMIT), (1, 2 + SMALL_LIMIT), (G // 2 + 3, G // 2 + 4), (G // 3, G // 3)]
    if G > 65536:
        b[4] = (8 * 4097, 8 * 4098)     # one 8-GPU node at an odd node index
    out = []
    for lo, hi in b:
        lo, hi = min(lo, G), min(hi, G)
        if (lo, hi) not in out:
            out.append((lo, hi))
    return out


SHAPES = [("few", 8), ("small", 40), ("small", 700), ("scan", 5000), ("spec", 6000), ("plain", 6000), ("chunks", 6000)]
RANGE_CASES = [(4096, 1, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT), (4096, 1, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT),
               (4096, 3, E.POLICY_FIRST_FIT, E.QUIRKS_FIXED), (4096, 3, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT),
               (65536, 1, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT), (65536, 1, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_FIXED),
               (65536, 3, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT), (65536, 3, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT),
               (300000, 1, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT), (300000, 1, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT)]


@pytest.mark.parametrize("G,n_tables,policy,quirks", RANGE_CASES)
def test_place_batch_range_paths(G, n_tables, policy, quirks):
    rng = W.SplitMix64(G + 10 * n_tables + 100 * policy + quirks)
    node_off = W.node_offsets(G // 8, 8)
    rows, node_table, n_names = tables_for(n_tables, G // 8, rng)
    occ = random_occ(rng, G)
    eng = make_engine(node_off, rows, occ, policy, quirks, node_table)
    chunk_eng = make_engine(node_off, rows, occ, policy, quirks, node_table, flags=E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL)
    whole = oracle.Fast(node_off, rows, quirks, policy, node_table=node_table)
    single = 0                          # 1g.10gb (H100) / the first name of the cluster: one placeable profile, scan mode
    scan_placed = 0
    for bi, (lo, hi) in enumerate(range_bounds(G)):
        occ = random_occ(rng, G)
        load(eng, node_off, occ, node_table)
        shapes = SHAPES + ([("two_chunks", 65537)] if bi < 3 else [])
        for shape, n in shapes:
            req = mixed_requests(rng, occ, lo, hi, n_names, n, profile=single if shape == "scan" else None)
            want, want_occ = place_range(node_off, rows, occ, lo, hi, req, quirks, policy, node_table)
            runs = [("", eng)]
            if shape == "few":
                runs = [("", eng), ("1", eng)]
            if shape == "chunks":
                chunk_eng.write_occupancy(0, occ)
                runs = [("", chunk_eng)]
            for no_few, e in runs:
                if len(runs) == 2 and no_few:
                    eng.write_occupancy(0, occ)         # the same call again, through k_small
                    os.environ["ISL_NO_FEW"] = "1"
                e.set_speculation(E.SPEC_OFF if shape == "plain" else E.SPEC_AUTO)
                what = (G, n_tables, policy, quirks, (lo, hi), shape, n, no_few)
                before = e.stats()
                try:
                    got = e.place_batch_range(lo, hi, req)
                finally:
                    os.environ.pop("ISL_NO_FEW", None)
                d = delta(e, before)
                compare(got, want, e.read_occupancy(), want_occ, what)
                path = {"few": "one", "small": "one", "two_chunks": "spec"}.get(shape, shape)
                check_path(d, path, n, what, G, lo, hi, n_tables)
                scan_placed += d["scan_placed"]
            if shape == "chunks":
                eng.write_occupancy(0, want_occ)
            occ = want_occ
        # the restriction is gone after the call: a whole-inventory batch lands anywhere
        req = mixed_requests(rng, occ, 0, G, n_names, 40)
        whole.load(occ)
        want = whole.place(req)
        compare(eng.place_batch(req), want, eng.read_occupancy(), whole.occupancy(), (G, (lo, hi), "whole"))
    assert scan_placed > 0          # the single-profile batches did commit through the capacity scan
    eng.close()
    chunk_eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG])
@pytest.mark.parametrize("n_tables", [1, 3])
def test_best_fit_family_on_ranges(policy, n_tables):
    """k_bestfit indexes occ[lo + g] and sizes its class bitmaps from hi - lo: shared memory up to 4096 GPUs of one table, global memory
    beyond that or with several tables."""
    G = 8192
    rng = W.SplitMix64(60 + policy + n_tables)
    node_off = W.node_offsets(G // 8, 8)
    rows, node_table, n_names = tables_for(n_tables, G // 8, rng)
    occ = random_occ(rng, G)
    eng = make_engine(node_off, rows, occ, policy, E.QUIRKS_REF_EXACT, node_table)
    n = 300 if policy == E.POLICY_MIN_FRAG else 1500
    for lo, hi in [(3, 19), (513, 4099), (4095, 8191), (1, G - 1), (4097, 4098), (77, 77)]:
        req = mixed_requests(rng, occ, lo, hi, n_names, n)
        want, want_occ = place_range(node_off, rows, occ, lo, hi, req, E.QUIRKS_REF_EXACT, policy, node_table)
        before = eng.stats()
        got = eng.place_batch_range(lo, hi, req)
        what = (policy, n_tables, (lo, hi))
        compare(got, want, eng.read_occupancy(), want_occ, what)
        check_path(delta(eng, before), "bestfit", n, what, G, lo, hi)
        occ = want_occ
    eng.close()


# ---- (b) isl_set_partition on one engine at unaligned bounds: every entry point ----------------------------------------------------------
PARTITIONS = [(65536, 13, 65536 - 29), (100000, 4097, 70001)]


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
@pytest.mark.parametrize("G,lo,hi", PARTITIONS)
def test_partition_entry_points(G, lo, hi, policy):
    import torch
    quirks = E.QUIRKS_REF_EXACT
    rng = W.SplitMix64(G + lo + policy)
    node_off = W.node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    n_names = len(rows)
    occ = random_occ(rng, G)
    eng = make_engine(node_off, rows, occ, policy, quirks, max_batch=4 * 65536)
    eng.set_partition(lo, hi)
    ref = RangeFast(node_off, rows, occ, lo, hi, quirks, policy)

    def place(e, req, path, n, what):
        before = e.stats()
        want = ref.place(req)
        got = e.place_batch(req)
        compare(got, want, e.read_occupancy(), ref.occupancy(), what)
        check_path(delta(e, before), path, n, what, G, lo, hi)

    # place_batch on every path
    for shape, n in SHAPES[:-1] + [("two_chunks", 65537)]:
        req = mixed_requests(rng, ref.occupancy(), lo, hi, n_names, n, profile=0 if shape == "scan" else None)
        eng.set_speculation(E.SPEC_OFF if shape == "plain" else E.SPEC_AUTO)
        place(eng, req, {"few": "one", "small": "one", "two_chunks": "spec"}.get(shape, shape), n, ("batch", shape, n))
    eng.set_speculation(E.SPEC_AUTO)
    # place_stream from pinned buffers: no causal window (plain pipeline, copier CTA), then window 1 (speculative rounds)
    for window in (0, 1):
        occ_now = ref.occupancy()
        batches = [mixed_requests(rng, occ_now, lo, hi, n_names, k) for k in (3000, 9000, 2000)]
        sizes = np.array([len(b) for b in batches], dtype=np.uint32)
        h_in, h_out = E.PinnedArray(int(sizes.sum()), E.REQUEST_DTYPE), E.PinnedArray(int(sizes.sum()), E.RESULT_DTYPE)
        h_in.array[:] = np.concatenate(batches)
        eng.set_causal_window(window)
        eng.place_stream_ptr(sizes, h_in.ptr, h_out.ptr, device=False)
        want = np.concatenate([ref.place(b) for b in batches])
        compare(h_out.array.copy(), want, eng.read_occupancy(), ref.occupancy(), ("stream", window))
        h_in.free(); h_out.free()
    eng.set_causal_window(0)
    # place_stream_device
    batches = [mixed_requests(rng, ref.occupancy(), lo, hi, n_names, k) for k in (5000, 700)]
    sizes = np.array([len(b) for b in batches], dtype=np.uint32)
    d_in = torch.from_numpy(np.concatenate(batches).view(np.uint8).copy()).cuda()
    d_out = torch.zeros(int(sizes.sum()) * 8, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    eng.place_stream_ptr(sizes, d_in.data_ptr(), d_out.data_ptr(), device=True)
    eng.synchronize()
    want = np.concatenate([ref.place(b) for b in batches])
    compare(d_out.cpu().numpy().view(E.RESULT_DTYPE), want, eng.read_occupancy(), ref.occupancy(), "stream_device")
    # an open stream, batch by batch
    n_batches, n = 3, 6000
    h_in, h_out = E.PinnedArray(n_batches * n, E.REQUEST_DTYPE), E.PinnedArray(n_batches * n, E.RESULT_DTYPE)
    eng.stream_open(n_batches)
    try:
        for b in range(n_batches):
            req = mixed_requests(rng, ref.occupancy(), lo, hi, n_names, n)
            h_in.array[b * n:(b + 1) * n] = req
            eng.stream_wait(eng.stream_submit_ptr(n, h_in.ptr + 8 * b * n, h_out.ptr + 8 * b * n))
            got, want = h_out.array[b * n:(b + 1) * n].copy(), ref.place(req)
            bad = np.flatnonzero(got != want)
            assert len(bad) == 0, ("open", b, bad[:5], got[bad[:5]], want[bad[:5]])
    finally:
        eng.stream_close()
    assert np.array_equal(eng.read_occupancy(), ref.occupancy()), "open stream"
    h_in.free(); h_out.free()
    # capacity over the slice
    occ_now = ref.occupancy()
    assert np.array_equal(eng.capacity(), capacity_by_hand(rows, quirks, occ_now[lo:hi])), "capacity"
    # what_if: records and capacities over the slice, the whole occupancy restored
    plan = mixed_requests(rng, occ_now, lo, hi, n_names, 3000)
    hypo = RangeFast(node_off, rows, occ_now, lo, hi, quirks, policy)
    want = hypo.place(plan)
    got, cap_before, cap_after = eng.what_if(plan)
    assert np.array_equal(got, want), "what_if"
    assert np.array_equal(cap_before, capacity_by_hand(rows, quirks, occ_now[lo:hi])), "what_if before"
    assert np.array_equal(cap_after, capacity_by_hand(rows, quirks, hypo.occupancy()[lo:hi])), "what_if after"
    assert np.array_equal(eng.read_occupancy(), occ_now), "what_if restore"
    # free_batch: spans inside the partition are released, outside ones and malformed ones are not
    gpus = np.r_[rng.next(200) % np.uint64(G), [lo, hi - 1, lo - 1, hi, G, G + 5]].astype(np.int64)
    spans = np.zeros(len(gpus), dtype=E.SPAN_DTYPE)
    expect = occ_now.copy()
    for i, g in enumerate(gpus):
        s, z = (0, 8) if g >= G else (int(rng.next1() % 4), 1 + int(rng.next1() % 4))
        spans[i] = (g, s, z, 0)
        if lo <= g < hi:
            expect[g] &= ~np.uint8(((1 << z) - 1) << s)
    eng.free_batch(spans)
    assert np.array_equal(eng.read_occupancy(), expect), "free_batch"
    ref = RangeFast(node_off, rows, expect, lo, hi, quirks, policy)
    # gangs, first-fit (this engine) and best-fit (a second engine with the same partition)
    for gang_policy in (policy, E.POLICY_BEST_FIT):
        e = eng if gang_policy == policy else make_engine(node_off, rows, ref.occupancy(), gang_policy, quirks)
        e.set_partition(lo, hi)
        gref = ref if gang_policy == policy else RangeFast(node_off, rows, ref.occupancy(), lo, hi, quirks, gang_policy)
        req = mixed_requests(rng, gref.occupancy(), lo, hi, n_names, 1200)
        cuts = (rng.next(300) % np.uint64(len(req))).astype(np.int64)
        off = np.unique(np.r_[0, cuts, len(req)]).astype(np.uint32)        # gangs of 1..~20 members
        want = GO.fast_place_gangs(gref, req, off, GO.default_sizes(rows))
        got = e.place_gangs(req, off)
        compare(got, want, e.read_occupancy(), gref.occupancy(), ("gangs", gang_policy))
        if e is not eng:
            e.close()
    eng.close()


# ---- (c) ISL_FLAG_ALL_NODES beyond k_small: unequal nodes, several 64-GPU segments per node -----------------------------------------
@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_all_nodes_unequal_nodes(policy):
    node_off = np.cumsum([0, 1, 7, 8, 13, 520, 600]).astype(np.uint32)
    G = int(node_off[-1])
    rng = W.SplitMix64(1149 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    occ = random_occ(rng, G)
    eng = make_engine(node_off, rows, occ, policy, E.QUIRKS_REF_EXACT, flags=E.FLAG_ALL_NODES)
    for lo, hi in [(0, G), (4, G - 300)]:           # the second cuts the 7-GPU node and the 600-GPU node in the middle
        for profile in (None, 0, None):
            req = mixed_requests(rng, occ, lo, hi, len(rows), 5000, profile=profile)
            want, want_occ = place_range(node_off, rows, occ, lo, hi, req, E.QUIRKS_REF_EXACT, policy, all_nodes=True)
            got = eng.place_batch(req) if (lo, hi) == (0, G) else eng.place_batch_range(lo, hi, req)
            compare(got, want, eng.read_occupancy(), want_occ, (policy, (lo, hi), profile))
            occ = want_occ
    eng.close()


# ---- (d) limits ---------------------------------------------------------------------------------------------------------------------------
def test_gang_and_best_fit_range_limit():
    """k_bestfit's class bitmaps cover at most 2^20 GPUs: a gang call on a larger partition and a best-fit engine for a larger inventory
    return ISL_ERANGE."""
    G = (1 << 20) + 1
    rows = E.make_profiles(tables.H100_80GB)
    eng = make_engine(W.node_offsets(G, 1), rows, np.zeros(G, dtype=np.uint8), E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT)
    eng.set_partition(0, G)
    req = W.alloc_requests(np.zeros(4, dtype=np.uint8))
    with pytest.raises(E.EngineError) as err:
        eng.place_gangs(req, [0, 2, 4])
    assert err.value.code == E.ERANGE
    eng.set_partition(0, G - 1)
    got = eng.place_gangs(req, [0, 2, 4])
    assert [(int(r["gpu"]), int(r["start"])) for r in got] == [(0, 0), (0, 1), (0, 2), (0, 3)]
    eng.close()
    with pytest.raises(E.EngineError) as err:
        E.Engine(max_gpus=G, max_batch=16, policy=E.POLICY_BEST_FIT)
    assert err.value.code == E.ERANGE


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG])
def test_empty_partition_on_every_entry_point(policy):
    """An empty partition: ALLOCs NO_CAPACITY, valid FREEs FREED and not applied, the occupancy unchanged, zero capacity; gangs ERANGE."""
    G, g = 4096, 1234
    rng = W.SplitMix64(4 + policy)
    node_off = W.node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ = random_occ(rng, G)
    eng = make_engine(node_off, rows, occ, policy, E.QUIRKS_REF_EXACT)
    eng.set_partition(g, g)
    for n in (8, 700, 6000, 65537):
        req = mixed_requests(rng, occ, g, g, len(rows), n)
        want, _ = place_range(node_off, rows, occ, g, g, req, E.QUIRKS_REF_EXACT, policy)
        assert not (want["status"] == E.ST_PLACED).any()
        compare(eng.place_batch(req), want, eng.read_occupancy(), occ, ("batch", n))
        compare(np.concatenate(eng.place_stream([req[: n // 2], req[n // 2:]])), want, eng.read_occupancy(), occ, ("stream", n))
        got, before, after = eng.what_if(req)
        assert np.array_equal(got, want) and not before.any() and not after.any(), ("what_if", n)
    assert not eng.capacity().any()
    eng.free_batch(np.array([(g, 0, 8, 0), (0, 0, 8, 0)], dtype=E.SPAN_DTYPE))
    assert np.array_equal(eng.read_occupancy(), occ)
    with pytest.raises(E.EngineError) as err:
        eng.place_gangs(W.alloc_requests(np.zeros(2, dtype=np.uint8)), [0, 2])
    assert err.value.code == E.ERANGE
    eng.close()
