"""Every device path at the limits of the profile-table ABI: 16 profile names, 8 node tables, 8 starts per row, 128 candidates (the
fixtures and their self-checks are in ``test_oracle_table_limits.py``).  Every call is compared with ``oracle.Fast`` byte for byte —
results and final occupancy — and the engine's counters show that the intended path ran.  Needs an H100.

Which test launches which k_pipeline<K, P15 = true, Spec> instantiation (16 profiles select P15):
  K = 1  T16mix-1   test_pipeline_with_16_profiles[*-t16mix1-*]       Spec = false with SPEC_OFF, true with SPEC_ON
  K = 2  T16mix-2   test_pipeline_with_16_profiles[*-t16mix2-*]
  K = 4  T16x8      test_pipeline_with_16_profiles[*-t16x8-*], test_edge65535_on_every_path, test_open_stream_t16x8,
                    test_plan_boundaries_for_128_candidates, test_partitioned_speculative_ring_t16x8; T8tab: test_t8tab_fixed_*
"""
import os

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W
from range_oracle import capacity_by_hand
from test_oracle_table_limits import (EDGE_N, candidates, churn_batches, default_sizes, edge65535, plus_one_candidate, ragged_nodes,
                                      t16mix, t16top, t16x8, t8tab, t8tab_node_tables)

pytestmark = pytest.mark.gpu


def make_engine(rows, node_off, occ, quirks, node_table=None, policy=E.POLICY_FIRST_FIT, flags=0, spec=None, max_batch=1 << 17):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, quirks=quirks, policy=policy, flags=flags)
    if spec is not None:
        eng.set_speculation(spec)
    if rows.ndim == 2:
        eng.load_profile_tables(rows)
    else:
        eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def make_oracle(rows, node_off, occ, quirks, node_table=None, policy=E.POLICY_FIRST_FIT):
    ref = oracle.Fast(node_off, rows, quirks, policy=policy, node_table=node_table)
    ref.load(occ)
    return ref


def check_batches(eng, batches, final, what):
    """place_batch of every (requests, oracle results) pair, then the final occupancy.  Returns the counters the calls added."""
    before = eng.stats()
    for i, (req, want) in enumerate(batches):
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (what, i, bad[:5], got[bad[:5]], want[bad[:5]], req[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), final), what
    after = eng.stats()
    return {k: after[k] - before[k] for k in ("kernel_launches", "spec_chunks", "scan_placed", "placed")}


def check_stream(eng, batches, final, what):
    got = eng.place_stream([req for req, _ in batches])
    for i, (g, (req, want)) in enumerate(zip(got, batches)):
        bad = np.flatnonzero(g != want)
        assert len(bad) == 0, (what, i, bad[:5], g[bad[:5]], want[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), final), what


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- k_few (<= 8 requests) and k_small (ISL_NO_FEW=1) --------------------------------------------------------------------------------
@pytest.mark.parametrize("name,quirks", [("t16mix1", q) for q in (0, 1, 2, 3)] + [("t16mix2", q) for q in (0, 1, 2, 3)] +
                         [("t8tab", 0), ("t8tab", 3), ("t16x8", 3)])
def test_few_and_small_paths(name, quirks):
    rows = {"t16mix1": lambda: t16mix(1), "t16mix2": lambda: t16mix(2), "t8tab": t8tab, "t16x8": t16x8}[name]()
    rng = W.SplitMix64(700 + quirks + 10 * len(name))
    n_nodes = 300
    node_off = ragged_nodes(rng, n_nodes)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes) if rows.ndim == 2 else None
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    occ[: G - 60] |= 0xFE                                       # nearly full: the search walks far
    ref = make_oracle(rows, node_off, occ, quirks, node_table)
    batches = churn_batches(rng, ref, [1 + int(rng.next1() % 8) for _ in range(120)], rows.shape[-1])
    for no_few in ("", "1"):
        os.environ.pop("ISL_NO_FEW", None)
        if no_few:
            os.environ["ISL_NO_FEW"] = "1"
        try:
            eng = make_engine(rows, node_off, occ, quirks, node_table)
            d = check_batches(eng, batches, ref.occupancy(), (name, quirks, no_few))
            assert d["kernel_launches"] == len(batches) and d["spec_chunks"] == 0, d         # one k_few / k_small launch per batch
            eng.close()
        finally:
            os.environ.pop("ISL_NO_FEW", None)


# ---- the chunk-by-chunk path: k_prepare, k_partition, sweeps, k_chain<K>, k_commit ----------------------------------------------------
@pytest.mark.parametrize("name,quirks", [("t16x8", 3), ("t16x8", 0), ("t8tab", 0)])
def test_chunk_path(name, quirks):
    rows = t16x8() if name == "t16x8" else t8tab()
    assert len(candidates(rows, quirks)) == 128                 # k_chain<4>
    rng = W.SplitMix64(800 + quirks + len(name))
    n_nodes = 600
    node_off = ragged_nodes(rng, n_nodes)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes) if rows.ndim == 2 else None
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    ref = make_oracle(rows, node_off, occ, quirks, node_table)
    batches = churn_batches(rng, ref, [900, 20_000, 70_000], 16)
    eng = make_engine(rows, node_off, occ, quirks, node_table, flags=E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL)
    d = check_batches(eng, batches, ref.occupancy(), name)
    assert d["kernel_launches"] == 3 + 5 * 4 and d["spec_chunks"] == 0, d        # k_prepare per batch; per chunk k_partition, two sweeps, k_chain, k_commit
    # a batch of profile 15 alone on the fresh inventory: the capacity scan commits it without a chain
    if rows.ndim == 1:
        eng.load_inventory(node_off, occ)
        ref = make_oracle(rows, node_off, occ, quirks)
        req = W.alloc_requests(np.full(5000, 15, dtype=np.uint8))
        d = check_batches(eng, [(req, ref.place(req))], ref.occupancy(), "scan")
        assert d["scan_placed"] == d["placed"] > 0, d
    eng.close()


# ---- the segment pipeline, plain and with speculative rounds, every K with 16 profiles ---------------------------------------------
PIPE_CASES = [("t16mix1", q) for q in (0, 1, 2, 3)] + [("t16mix2", q) for q in (0, 1, 2, 3)] + [("t16x8", 3), ("t16x8", 0)]


@pytest.mark.parametrize("spec", [E.SPEC_OFF, E.SPEC_ON])
@pytest.mark.parametrize("name,quirks", PIPE_CASES)
def test_pipeline_with_16_profiles(name, quirks, spec):
    """k_pipeline<K, true, Spec>: single batches with frees through FLAG_FORCE_PIPELINE, then a churn stream with a causal window of 1."""
    rows = {"t16mix1": lambda: t16mix(1), "t16mix2": lambda: t16mix(2), "t16x8": t16x8}[name]()
    rng = W.SplitMix64(900 + 4 * quirks + spec + 10 * len(name))
    n_nodes = 500
    node_off = ragged_nodes(rng, n_nodes)
    G = int(node_off[-1])
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    ref = make_oracle(rows, node_off, occ, quirks)
    batches = churn_batches(rng, ref, [3000, 70_000, 9000], 16)
    eng = make_engine(rows, node_off, occ, quirks, flags=E.FLAG_FORCE_PIPELINE, spec=spec)
    d = check_batches(eng, batches, ref.occupancy(), (name, quirks, spec))
    assert d["kernel_launches"] == 3 * len(batches), d                             # k_prepare + k_partition + ONE k_pipeline per batch
    assert (d["spec_chunks"] == 4) if spec == E.SPEC_ON else (d["spec_chunks"] == 0), d
    # a churn stream, each batch composed from the results of the one before, with a causal window of 1
    eng.load_inventory(node_off, occ)
    ref = make_oracle(rows, node_off, occ, quirks)
    stream = churn_batches(rng, ref, [6000] * 6, 16, frees=2)
    eng.set_causal_window(1)
    before = eng.stats()["spec_chunks"]
    check_stream(eng, stream, ref.occupancy(), (name, quirks, spec, "stream"))
    assert (eng.stats()["spec_chunks"] - before == 6) if spec == E.SPEC_ON else (eng.stats()["spec_chunks"] == before)
    eng.close()


@pytest.mark.parametrize("path", ["spec", "plain", "chunks"])
def test_edge65535_on_every_path(path):
    """The last request of a full chunk is profile 15 (key bits 11..30 all set) and is placed while other lanes are exhausted."""
    rows = t16x8()
    node_off, occ, req = edge65535(W.SplitMix64(65535))
    ref = make_oracle(rows, node_off, occ, E.QUIRKS_REF_EXACT)
    want = ref.place(req)
    assert want["status"][EDGE_N - 1] == E.ST_PLACED
    flags = E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL if path == "chunks" else E.FLAG_FORCE_PIPELINE
    eng = make_engine(rows, node_off, occ, E.QUIRKS_REF_EXACT, flags=flags, spec=E.SPEC_ON if path == "spec" else E.SPEC_OFF)
    d = check_batches(eng, [(req, want)], ref.occupancy(), path)
    assert d["spec_chunks"] == (1 if path == "spec" else 0), d
    assert d["kernel_launches"] == (6 if path == "chunks" else 3), d
    eng.close()


@pytest.mark.parametrize("spec", [E.SPEC_ON, E.SPEC_OFF])
def test_t8tab_fixed_quirks_on_the_pipeline(spec):
    """8 tables, more than 32 candidates of >= 4 slices (the speculative prologue keeps 32), odd sizes: rounds may cost more, never
    exactness."""
    rows = t8tab()
    rng = W.SplitMix64(88 + spec)
    n_nodes = 700
    node_off = ragged_nodes(rng, n_nodes)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes)
    occ = ((rng.next(G) & rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    ref = make_oracle(rows, node_off, occ, E.QUIRKS_FIXED, node_table)
    batches = churn_batches(rng, ref, [2000, 40_000, 70_000, 500], 16)
    eng = make_engine(rows, node_off, occ, E.QUIRKS_FIXED, node_table, flags=E.FLAG_FORCE_PIPELINE, spec=spec)
    d = check_batches(eng, batches, ref.occupancy(), spec)
    assert (d["spec_chunks"] == 5) if spec == E.SPEC_ON else (d["spec_chunks"] == 0), d
    # the same batches as one stream with a causal window of 1 on a fresh inventory
    eng.load_inventory(node_off, occ)
    eng.set_node_tables(node_table)
    eng.set_causal_window(1)
    check_stream(eng, batches, ref.occupancy(), (spec, "stream"))
    eng.close()


@pytest.mark.parametrize("spec", [E.SPEC_ON, E.SPEC_OFF])
def test_open_stream_t16x8(spec):
    rows = t16x8()
    G, n, n_batches = 4096, 8000, 5
    rng = W.SplitMix64(4242 + spec)
    node_off = W.node_offsets(G // 8, 8)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    ref = make_oracle(rows, node_off, occ, E.QUIRKS_REF_EXACT)
    eng = make_engine(rows, node_off, occ, E.QUIRKS_REF_EXACT, spec=spec, max_batch=n_batches * 65536)
    h_in = E.PinnedArray(n_batches * n, E.REQUEST_DTYPE)
    h_out = E.PinnedArray(n_batches * n, E.RESULT_DTYPE)
    eng.stream_open(n_batches)
    live = []
    for b in range(n_batches):          # strictly causal: batch b is composed from the results of batch b - 1
        req = W.alloc_requests((rng.next(n) % np.uint64(16)).astype(np.uint8))
        for _ in range(min(len(live), n // 2)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        h_in.array[b * n:(b + 1) * n] = req
        t = eng.stream_submit_ptr(n, h_in.ptr + 8 * b * n, h_out.ptr + 8 * b * n)
        eng.stream_wait(t)
        got = h_out.array[b * n:(b + 1) * n].copy()
        want = ref.place(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (b, bad[:5], got[bad[:5]], want[bad[:5]])
        live.extend((int(r["gpu"]), int(r["start"]), int(r["size"])) for r in got[(req["op"] == E.OP_ALLOC) & (got["status"] == E.ST_PLACED)])
    eng.stream_close()
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    st = eng.stats()
    assert (st["spec_chunks"] == n_batches) if spec == E.SPEC_ON else (st["spec_chunks"] == 0), st
    h_in.free(); h_out.free()
    eng.close()


# ---- where the plan changes for 128 candidates: 64-GPU segments, from the SM count ------------------------------------------------
def test_plan_boundaries_for_128_candidates():
    """128 candidates cap a (sub-)segment at 64 GPUs (max_segment_for).  One batch gets speculative rounds while every SM's stage is one
    64-GPU segment (SMs x 64 GPUs), a plain pipeline of up to 8 sub-segments per stage beyond that (SMs x 8 x 64 GPUs), and the
    chunk-by-chunk path beyond that."""
    rows = t16x8()
    sms = sm_count()
    cases = [(sms * 64, "spec"), (sms * 64 + 64, "plain"), (sms * 8 * 64, "plain"), (sms * 8 * 64 + 64, "chunks")]
    rng = W.SplitMix64(128)
    for G, path in cases:
        node_off = W.node_offsets(G // 8, 8)
        occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
        ref = make_oracle(rows, node_off, occ, E.QUIRKS_REF_EXACT)
        req = W.alloc_requests((rng.next(20_000) % np.uint64(16)).astype(np.uint8))       # mixed: the pipeline is the default route
        eng = make_engine(rows, node_off, occ, E.QUIRKS_REF_EXACT, spec=E.SPEC_ON)
        d = check_batches(eng, [(req, ref.place(req))], ref.occupancy(), (G, path))
        assert d["spec_chunks"] == (1 if path == "spec" else 0), (G, path, d)
        assert d["kernel_launches"] == (6 if path == "chunks" else 3), (G, path, d)
        eng.close()


def test_partitioned_speculative_ring_t16x8():
    """Two engines on one GPU, each owning half of the inventory, their record memories wired into each other: the stages of both form
    one speculative sequence; the owner's result array == the global sequential first-fit."""
    import torch
    from instaslice_b200 import dist as D
    n_ranks, window = 2, 1
    rows = t16x8()
    rng = W.SplitMix64(2024)
    G = 4096
    node_off = W.node_offsets(G // 8, 8)
    occ0 = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    ref = make_oracle(rows, node_off, occ0, E.QUIRKS_REF_EXACT)
    batches = churn_batches(rng, ref, [3000 + 700 * b for b in range(5)], 16)
    want = [res for _, res in batches]
    sizes = np.array([len(req) for req, _ in batches], dtype=np.uint32)
    n_ops = int(sizes.sum())
    d_in = torch.from_numpy(np.concatenate([req for req, _ in batches]).view(np.int64).copy()).cuda()
    bounds = D.all_bounds(G, n_ranks, align=64)
    cuts = [lo for lo, _ in bounds] + [G]
    engines = []
    for lo, hi in bounds:
        eng = make_engine(rows, node_off, occ0, E.QUIRKS_REF_EXACT, max_batch=1 << 16)
        eng.ipc_inbox_handle(); eng.ipc_spec_handle()          # allocate the shared buffers
        engines.append(eng)
    for r, eng in enumerate(engines):
        eng.connect_local(engines[r + 1] if r + 1 < n_ranks else None, has_prev=r > 0)
        eng.connect_owner_local(engines[0] if r > 0 else None)
        eng.set_ring_world(n_ranks)
        eng.connect_spec_local(n_ranks, r, engines, cuts)
        eng.set_causal_window(window)
        eng.set_speculation(E.SPEC_ON)
    torch.cuda.synchronize()
    for stream_id in (1, 2):
        for eng, (lo, hi) in zip(engines, bounds):
            eng.load_inventory(node_off, occ0)
            eng.set_partition(lo, hi)
        for eng in engines:
            eng.place_stream_partitioned(sizes, d_in.data_ptr(), eng.device_results(), stream_id)
        for eng in engines:
            eng.synchronize()

        class _View:            # torch view of the owner's engine-owned result array (no copy)
            __cuda_array_interface__ = {"shape": (n_ops,), "typestr": "<i8", "data": (engines[0].device_results(), False), "version": 3}
        got = torch.as_tensor(_View(), device="cuda").cpu().numpy().view(E.RESULT_DTYPE)
        bad = np.flatnonzero(got != np.concatenate(want))
        assert len(bad) == 0, (stream_id, bad[:5])
        occ = np.concatenate([eng.read_occupancy()[lo:hi] for eng, (lo, hi) in zip(engines, bounds)])
        assert np.array_equal(occ, ref.occupancy())
        assert engines[-1].stats()["spec_chunks"] >= len(batches)
    for eng in engines:
        eng.close()


# ---- allocation policies ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy,name,quirks", [(E.POLICY_BEST_FIT, "t16x8", 3), (E.POLICY_MIN_FRAG, "t16x8", 3),
                                                (E.POLICY_BEST_FIT, "t16mix2", 0), (E.POLICY_MIN_FRAG, "t16mix2", 0),
                                                (E.POLICY_MIN_FRAG, "t16top", 0),
                                                (E.POLICY_BEST_FIT, "t8tab", 0), (E.POLICY_MIN_FRAG, "t8tab", 0),
                                                (E.POLICY_RIGHT_TO_LEFT, "t8tab", 0)])
def test_policies(policy, name, quirks):
    rows = {"t16x8": t16x8, "t16mix2": lambda: t16mix(2), "t16top": t16top, "t8tab": t8tab}[name]()
    rng = W.SplitMix64(60 + policy + len(name))
    n_nodes = 400
    node_off = ragged_nodes(rng, n_nodes)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes) if rows.ndim == 2 else None
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    occ[rng.next(G) % np.uint64(7) == 0] = 0                  # empty GPUs: where a size-8 row scores its 121
    ref = make_oracle(rows, node_off, occ, quirks, node_table, policy)
    sizes = [7, 300, 1500] if policy != E.POLICY_RIGHT_TO_LEFT else [3, 1, 700, 5000, 70_000, 8, 1500]
    batches = churn_batches(rng, ref, sizes, 16)
    eng = make_engine(rows, node_off, occ, quirks, node_table, policy=policy)
    check_batches(eng, batches, ref.occupancy(), (policy, name))
    if policy == E.POLICY_RIGHT_TO_LEFT:        # and as one stream through the segment pipeline
        eng.load_inventory(node_off, occ)
        eng.set_node_tables(node_table)
        check_stream(eng, batches, ref.occupancy(), "stream")
    eng.close()


# ---- queries ------------------------------------------------------------------------------------------------------------------------
def test_capacity_and_what_if_t8tab():
    rows = t8tab()
    rng = W.SplitMix64(31337)
    n_nodes = 500
    node_off = ragged_nodes(rng, n_nodes)
    G = int(node_off[-1])
    node_table = t8tab_node_tables(rng, n_nodes)
    gpu_table = np.repeat(node_table, np.diff(node_off))
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
    eng = make_engine(rows, node_off, occ, E.QUIRKS_FIXED, node_table)
    assert np.array_equal(eng.capacity(), capacity_by_hand(rows, E.QUIRKS_FIXED, occ, gpu_table))
    ref = make_oracle(rows, node_off, occ, E.QUIRKS_FIXED, node_table)
    plan = W.alloc_requests((rng.next(3000) % np.uint64(16)).astype(np.uint8))
    for i, g in enumerate(np.flatnonzero(occ & 1)[:200]):        # release 200 busy slices first
        plan[i] = (g, 0, E.OP_FREE, 0, 1)
    want = ref.place(plan)
    got, before, after = eng.what_if(plan)
    assert np.array_equal(got, want)
    assert np.array_equal(before, capacity_by_hand(rows, E.QUIRKS_FIXED, occ, gpu_table))
    assert np.array_equal(after, capacity_by_hand(rows, E.QUIRKS_FIXED, ref.occupancy(), gpu_table))
    assert np.array_equal(eng.read_occupancy(), occ)            # the live state is back
    # an unplaced request reports the size of the first node (canonical order) whose table knows the name: table 7 for profile 15
    full = np.full(G, 0xFF, dtype=np.uint8)
    eng.load_inventory(node_off, full)
    eng.set_node_tables(node_table)
    res = eng.place_batch(W.alloc_requests(np.arange(16, dtype=np.uint8)))
    assert (res["status"] == E.ST_NO_CAPACITY).all() and res["size"].tolist() == default_sizes(rows, node_table)
    assert int(res["size"][15]) == int(rows["size"][7, 15])
    eng.close()


# ---- the ABI limits themselves -------------------------------------------------------------------------------------------------
def test_abi_limits_accepted_and_one_beyond_rejected():
    eng = E.Engine(max_gpus=4096, max_batch=1024, quirks=E.QUIRKS_FIXED)

    def code(fn, *args):
        try:
            fn(*args)
            return E.OK
        except E.EngineError as e:
            return e.code

    x8, tabs = t16x8(), t8tab()
    assert code(eng.load_profiles, x8) == E.OK                                  # 16 names, 8 starts, 128 candidates
    assert code(eng.load_profile_tables, tabs) == E.OK                          # 8 tables, 128 candidates
    seventeen = np.concatenate([x8, x8[:1]])
    assert code(eng.load_profiles, seventeen) == E.EINVAL
    assert code(eng.load_profile_tables, np.concatenate([tabs, tabs[:1]])) == E.EINVAL
    assert code(eng.load_profile_tables, plus_one_candidate(tabs, E.QUIRKS_FIXED)) == E.EINVAL
    nine = t16mix(1)
    nine["n_starts"][0] = 9                                                     # a 9th start
    assert code(eng.load_profiles, nine) == E.EINVAL
    # a rejected table leaves the loaded one in place: T8tab still places
    eng.load_inventory(W.node_offsets(4, 8), np.zeros(32, dtype=np.uint8))
    ref = make_oracle(tabs, W.node_offsets(4, 8), np.zeros(32, dtype=np.uint8), E.QUIRKS_FIXED, np.zeros(4, dtype=np.uint8))
    req = W.alloc_requests(np.arange(16, dtype=np.uint8))
    assert np.array_equal(eng.place_batch(req), ref.place(req))
    eng.close()
