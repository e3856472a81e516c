"""Parity of the CUDA engine (through the C ABI) against the oracle and the golden vectors.  Needs an H100.

Bar: bit-exact (integer / index work) — results AND final occupancy, byte for byte.
"""
import copy
import json
import os

import numpy as np
import pytest

import oracle
from oracle import ref_py
from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables, workloads as W

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    with open(os.path.join(GOLD, name)) as f:
        return json.load(f)


def make_engine(node_off, occ, rows, quirks=E.QUIRKS_REF_EXACT, max_batch=1 << 20, flags=0):
    eng = E.Engine(max_gpus=max(4096, len(occ)), max_batch=max_batch, quirks=quirks, flags=flags)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    return eng


def check_against_fast(node_off, occ, rows, batches, quirks=E.QUIRKS_REF_EXACT):
    """Every batch through both device paths (single chain, forced segment pipeline) and as ONE stream call."""
    ref = oracle.Fast(node_off, rows, quirks)
    ref.load(occ)
    want = [ref.place(req) for req in batches]
    final = ref.occupancy()
    for flags in (E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL, E.FLAG_FORCE_PIPELINE, 0):
        eng = make_engine(node_off, occ, rows, quirks, flags=flags)
        for i, req in enumerate(batches):
            got = eng.place_batch(req)
            bad = np.flatnonzero(got != want[i])
            assert len(bad) == 0, (flags, i, bad[:5], got[bad[:5]], want[i][bad[:5]], req[bad[:5]])
        assert np.array_equal(eng.read_occupancy(), final), flags
    eng = make_engine(node_off, occ, rows, quirks)
    got = eng.place_stream(batches)
    for i, (g, w) in enumerate(zip(got, want)):
        bad = np.flatnonzero(g != w)
        assert len(bad) == 0, ("stream", i, bad[:5], g[bad[:5]], w[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), final)
    return eng


# ---- the device table: every (occupancy byte, profile row), both tables, all quirk sets --------------------
@pytest.mark.parametrize("quirks", [3, 0, 1, 2])
@pytest.mark.parametrize("tname", ["a100-40gb", "h100-80gb", "a30-24gb", "b200-180gb"])
def test_device_table_exhaustive(tname, quirks):
    rows = E.make_profiles(tables.TABLES[tname])
    eng = E.Engine(max_gpus=4096, max_batch=1024, quirks=quirks)
    eng.load_profiles(rows)
    occ = np.arange(256, dtype=np.uint8)
    for p in range(len(rows)):
        got = eng.eval_starts(p, occ)
        want = np.array([oracle.start_for(rows[p], quirks, o) for o in range(256)], dtype=np.uint8)
        assert np.array_equal(got, want), (tname, quirks, p)


def test_device_table_odd_rows():
    """Rows NVML never emits but a CRD may hold: size 3/5/6/7, unordered starts, start+size > 8."""
    table = [("a", 3, [0, 3, 5], 0), ("b", 2, [6, 4, 1, 0], 1), ("c", 1, [7, 0], 2), ("d", 8, [0], 3), ("e", 4, [4, 3, 1], 4),
             ("f", 7, [1, 0], 5), ("g", 5, [3, 2], 6), ("h", 6, [2, 1, 0], 7)]
    rows = E.make_profiles(table)
    occ = np.arange(256, dtype=np.uint8)
    for quirks in (3, 0, 1, 2):
        eng = E.Engine(max_gpus=4096, max_batch=1024, quirks=quirks)
        eng.load_profiles(rows)
        for p in range(len(rows)):
            want = np.array([oracle.start_for(rows[p], quirks, o) for o in range(256)], dtype=np.uint8)
            assert np.array_equal(eng.eval_starts(p, occ), want), (quirks, p)


def test_kat_golden_on_device():
    kat = load("kat_starts.json")
    table = tables.TABLES[kat["table"]]
    eng = E.Engine(max_gpus=4096, max_batch=1024, quirks=kat["quirks"])
    eng.load_profiles(E.make_profiles(table))
    for occ_hex, want in kat["starts"].items():
        for col, name in enumerate(kat["profiles"]):
            got = eng.eval_starts(tables.profile_index(table, name), np.array([int(occ_hex, 16)], dtype=np.uint8))
            assert int(got[0]) == want[col], (occ_hex, name)


# ---- golden sequences and BASELINE configs ---------------------------------------------------------------
def test_golden_sequences():
    for case in load("sequences.json")["cases"]:
        table = tables.TABLES[case["table"]]
        rows = E.make_profiles(table)
        eng = make_engine(W.node_offsets(1, case["gpus"]), np.array(case["occ"], dtype=np.uint8), rows)
        req = W.alloc_requests(np.array([tables.profile_index(table, n) for n in case["profiles"]], dtype=np.uint8))
        res = eng.place_batch(req)
        assert res["start"].tolist() == case["start"], case["name"]
        assert [None if g == E.GPU_NONE else int(g) for g in res["gpu"]] == case["gpu"], case["name"]
        assert eng.read_occupancy().tolist() == case["final_occ"], case["name"]


def test_config1_through_controller_mirror():
    """samples/test-pod.yaml on one emulated A100-40GB GPU, through the reference-named interface."""
    case = [c for c in load("sequences.json")["cases"] if c["name"] == "config1_test_pod"][0]
    cr = {"metadata": {"name": "kind-control-plane"},
          "spec": {"MigGPUUUID": {"GPU-31cfe05c-ed13-cd17-d7aa-c63db5108c24": "NVIDIA A100-PCIE-40GB"},
                   "migplacement": tables.migplacement(tables.A100_40GB)}}
    r = ctl.InstasliceReconciler([cr])
    limits = {"nvidia.com/mig-1g.5gb": 1, "org.instaslice/cuda-vectoradd-1": 1}
    name = r.extractProfileName(limits)
    assert name == "1g.5gb"
    pod = {"uid": "uid-1", "name": "cuda-vectoradd-1", "namespace": "default"}
    alloc = r.findDeviceForASlice(cr, name, ctl.FirstFitPolicy(), pod)
    for key, val in case["allocation"].items():
        assert alloc[key] == val
    assert alloc["gpuUUID"].startswith("GPU-31cfe05c") and alloc["podUUID"] == "uid-1" and alloc["nodename"] == "kind-control-plane"
    assert r.getStartIndexFromPreparedState(cr, alloc["gpuUUID"], "7g.40gb") == 9        # Q1: 7g never places
    with pytest.raises(ctl.AllocationError, match="failed to find allocatable gpu"):
        r.findDeviceForASlice(cr, "7g.40gb", ctl.FirstFitPolicy(), pod)
    assert ctl.LeftToRightPolicy().SetAllocationDetails() == {}                        # the reference's stubs


def test_config2_closed_form():
    node_off, occ, rows, req = W.config2()
    eng = make_engine(node_off, occ, rows)
    res = eng.place_batch(req)
    k = np.arange(len(req))
    placed = k < 1792
    assert np.array_equal(res["status"] == E.ST_PLACED, placed)
    assert np.array_equal(res["gpu"][placed], (k[placed] // 7).astype(np.uint32))
    assert np.array_equal(res["start"][placed], (k[placed] % 7).astype(np.uint8))
    assert (res["start"][~placed] == 9).all() and (res["gpu"][~placed] == E.GPU_NONE).all() and (res["status"][~placed] == E.ST_NO_CAPACITY).all()
    assert (eng.read_occupancy() == 0x7F).all()


def test_config3_first_fit_vs_oracle():
    node_off, occ, rows, req = W.config3()
    check_against_fast(node_off, occ, rows, [req])          # 100k requests = 2 commit chunks in one call


def test_regress_crd_golden_through_controller_mirror():
    """Random CR states (dangling / allocated / realised / orphan slices, unknown profiles, veto), pod by pod."""
    gold = load("regress_crd.json")
    for ci, case in enumerate(gold["cases"]):
        items = copy.deepcopy(case["instaslices"])
        r = ctl.InstasliceReconciler(items, quirks=case["quirks"])
        for pod, want in zip(case["pods"], case["outcomes"]):
            verdict, alloc = r.reconcile_gated_pod({"uid": pod["uid"], "name": pod["uid"]}, pod["profile"])
            assert verdict == want["verdict"], (ci, pod)
            if alloc:
                assert (alloc["gpuUUID"], alloc["nodename"], alloc["start"], alloc["size"], alloc["giprofileid"]) == \
                       (want["gpuUUID"], want["nodename"], want["start"], want["size"], want["giprofileid"]), (ci, pod)


def test_regress_crd_batched_equals_pod_by_pod():
    gold = load("regress_crd.json")
    for case in gold["cases"]:
        items = copy.deepcopy(case["instaslices"])
        r = ctl.InstasliceReconciler(items, quirks=case["quirks"])
        pods = [{"uid": p["uid"], "name": p["uid"], "profile": p["profile"]} for p in case["pods"]]
        out = r.place_pending_pods(pods)
        assert [v for v, _ in out] == [w["verdict"] for w in case["outcomes"]]
        for (v, a), w in zip(out, case["outcomes"]):
            if a:
                assert (a["gpuUUID"], a["start"]) == (w["gpuUUID"], w["start"])


# ---- randomised parity, edge cases ------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL, E.FLAG_FORCE_PIPELINE, 0])
@pytest.mark.parametrize("quirks", [3, 0])
@pytest.mark.parametrize("tname", ["a100-40gb", "h100-80gb", "a30-24gb", "b200-180gb"])
def test_random_occupancy_and_frees(tname, quirks, flags):
    table = tables.TABLES[tname]
    rows = E.make_profiles(table)
    rng = W.SplitMix64(31 + quirks)
    for trial in range(4):
        n_nodes = 1 + int(rng.next1() % 700)
        node_off = np.concatenate([[0], np.cumsum(1 + (rng.next(n_nodes) % np.uint64(9)).astype(np.int64))]).astype(np.uint32)
        G = int(node_off[-1])
        occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
        eng = make_engine(node_off, occ, rows, quirks, flags=flags)
        ref = oracle.Fast(node_off, rows, quirks)
        ref.load(occ)
        live = []
        for batch in range(5):
            n = 1 + int(rng.next1() % 3000)
            req = W.alloc_requests((rng.next(n) % np.uint64(len(table) + 1)).astype(np.uint8))
            req["profile"][req["profile"] == len(table)] = E.PROFILE_UNKNOWN
            n_free = min(len(live), n // 3)
            for i in range(n_free):
                g, s, z = live.pop(int(rng.next1() % len(live)))
                req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
            got, want = eng.place_batch(req), ref.place(req)
            assert np.array_equal(got, want), (tname, quirks, trial, batch)
            assert np.array_equal(eng.read_occupancy(), ref.occupancy())
            for r in got[(req["op"] == E.OP_ALLOC) & (got["status"] == E.ST_PLACED)]:
                live.append((int(r["gpu"]), int(r["start"]), int(r["size"])))
            assert eng.gpu_to_node(G - 1) == n_nodes - 1 and eng.gpu_to_node(0) == 0


def test_edge_cases():
    rows = E.make_profiles(tables.H100_80GB)
    node_off = W.node_offsets(3, 2)
    eng = make_engine(node_off, np.zeros(6, dtype=np.uint8), rows)
    # empty batch
    assert len(eng.place_batch(np.zeros(0, dtype=E.REQUEST_DTYPE))) == 0
    # unknown profile, NOOP, bad spans
    req = np.zeros(6, dtype=E.REQUEST_DTYPE)
    req[0] = (0, E.PROFILE_UNKNOWN, E.OP_ALLOC, 0, 0)
    req[1] = (0, 0, E.OP_NOOP, 0, 0)
    req[2] = (99, 0, E.OP_FREE, 0, 1)        # GPU outside the inventory
    req[3] = (0, 0, E.OP_FREE, 6, 4)         # span beyond slice 7
    req[4] = (0, 0, E.OP_FREE, 0, 0)         # empty span
    req[5] = (0, 5, E.OP_ALLOC, 0, 0)        # 7g.80gb: never places under REF_EXACT (Q1)
    ref = oracle.Fast(node_off, rows)
    ref.load(np.zeros(6, dtype=np.uint8))
    want = ref.place(req)
    # every request pre-pass: k_few (default), k_small, k_prepare on the chunk path and in stream mode (free mask)
    for flags, no_few in ((0, ""), (0, "1"), (E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL, ""), (E.FLAG_FORCE_PIPELINE, "")):
        os.environ.pop("ISL_NO_FEW", None)
        if no_few:
            os.environ["ISL_NO_FEW"] = "1"
        try:
            path = make_engine(node_off, np.zeros(6, dtype=np.uint8), rows, flags=flags)
            res = path.place_batch(req)
        finally:
            os.environ.pop("ISL_NO_FEW", None)
        assert res["status"].tolist() == [E.ST_BAD_PROFILE, E.ST_NOOP, E.ST_BAD_SPAN, E.ST_BAD_SPAN, E.ST_BAD_SPAN, E.ST_NO_CAPACITY], (flags, no_few)
        assert (path.read_occupancy() == 0).all(), (flags, no_few)
        assert np.array_equal(res, want), (flags, no_few)
        path.close()
    # freeing a span and re-allocating it in the same batch: frees are applied first
    eng.place_batch(W.alloc_requests(np.array([4], dtype=np.uint8)))                    # 4g at gpu0:0-3
    req = np.zeros(2, dtype=E.REQUEST_DTYPE)
    req[0] = (0, 4, E.OP_ALLOC, 0, 0)
    req[1] = (0, 0, E.OP_FREE, 0, 4)
    res = eng.place_batch(req)
    assert (int(res["gpu"][0]), int(res["start"][0])) == (0, 0)
    # separate free entry point
    spans = np.zeros(1, dtype=E.SPAN_DTYPE)
    spans[0] = (0, 0, 4, 0)
    eng.free_batch(spans)
    assert eng.read_occupancy()[0] == 0
    # capacity errors
    with pytest.raises(E.EngineError) as ei:
        E.Engine(max_gpus=4096, max_batch=8).place_batch(np.zeros(1, dtype=E.REQUEST_DTYPE))
    assert ei.value.code == E.ESTATE
    small = make_engine(node_off, np.zeros(6, dtype=np.uint8), rows, max_batch=8)
    with pytest.raises(E.EngineError) as ei:
        small.place_batch(np.zeros(9, dtype=E.REQUEST_DTYPE))
    assert ei.value.code == E.ERANGE
    # malformed tables are rejected instead of panicking (Q7)
    bad = E.make_profiles([("x", 1, [0], 0)])
    bad[0]["starts"][0] = 8
    with pytest.raises(E.EngineError):
        small.load_profiles(bad)
    bad = E.make_profiles([("x", 1, [0], 0)])
    bad[0]["n_starts"] = 0
    with pytest.raises(E.EngineError):
        small.load_profiles(bad)


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 65535, 65536, 65537, 131072 + 5])
def test_chunk_and_tile_boundaries(n):
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(n)
    node_off = W.node_offsets(2048, 8)
    occ = ((rng.next(16384) & rng.next(16384)) & np.uint64(0x7F)).astype(np.uint8)
    check_against_fast(node_off, occ, rows, [W.alloc_requests(W.mix_profiles(rng, n))])


def test_single_profile_runs_and_exhaustion():
    """Long homogeneous runs and total exhaustion of the inventory."""
    rows = E.make_profiles(tables.H100_80GB)
    node_off = W.node_offsets(64, 8)
    prof = np.concatenate([np.full(3000, 4, np.uint8), np.full(3000, 2, np.uint8), np.full(5000, 0, np.uint8)])
    check_against_fast(node_off, np.zeros(512, dtype=np.uint8), rows, [W.alloc_requests(prof), W.alloc_requests(prof[::-1].copy())])


def test_many_candidate_table_uses_multi_slot_chain():
    """A table with more than 32 and more than 64 legal (profile, start) pairs (k_chain<2>, k_chain<4>)."""
    for n_rows in (6, 12):
        table = [("s%d" % i, 1 + (i % 2), [(j + i) % 7 for j in range(7)], i) for i in range(n_rows)]
        rows = E.make_profiles(table)
        rng = W.SplitMix64(n_rows)
        node_off = W.node_offsets(300, 8)
        occ = ((rng.next(2400) & rng.next(2400)) & np.uint64(0xFF)).astype(np.uint8)
        req = W.alloc_requests((rng.next(20000) % np.uint64(n_rows)).astype(np.uint8))
        check_against_fast(node_off, occ, rows, [req], quirks=0)


# ---- full-size runs: BASELINE config 4 shape, size-independent properties + oracle ----------------------------
def test_config4_churn_full_size():
    ch = W.Churn()                                   # 65 536 GPUs, 1M ops, batches of 65 536, seed 42
    eng = make_engine(ch.node_off, np.zeros(ch.G, dtype=np.uint8), ch.rows)
    results = []

    def placer(req):
        res = eng.place_batch(req)
        results.append(res)
        return res

    batches = ch.generate(placer)
    # property: no double booking — occupancy == union of live spans, and popcount == sum of live sizes
    occ = eng.read_occupancy()
    live = {}
    for req, res in zip(batches, results):
        fr = req["op"] == E.OP_FREE
        for g, s in zip(req["handle"][fr], req["start"][fr]):
            del live[(int(g), int(s))]
        pl = (req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)
        for g, s, z in zip(res["gpu"][pl], res["start"][pl], res["size"][pl]):
            assert (int(g), int(s)) not in live
            live[(int(g), int(s))] = int(z)
    rebuilt = np.zeros(ch.G, dtype=np.uint8)
    total = 0
    for (g, s), z in live.items():
        span = ((1 << z) - 1) << s
        assert rebuilt[g] & span == 0, "double booking"
        rebuilt[g] |= span
        total += z
    assert np.array_equal(rebuilt, occ)
    assert int(np.unpackbits(occ).sum()) == total
    # and byte-for-byte against the oracle on the same recorded batches
    ref = oracle.Fast(ch.node_off, ch.rows)
    ref.load(np.zeros(ch.G, dtype=np.uint8))
    for i, (req, res) in enumerate(zip(batches, results)):
        assert np.array_equal(ref.place(req), res), i
    assert np.array_equal(ref.occupancy(), occ)
    # replay is deterministic (idempotence of the recorded run)
    eng2 = make_engine(ch.node_off, np.zeros(ch.G, dtype=np.uint8), ch.rows)
    for req, res in zip(batches, results):
        assert np.array_equal(eng2.place_batch(req), res)
    # the whole recorded run as ONE stream call through the segment pipeline: identical, byte for byte
    eng3 = make_engine(ch.node_off, np.zeros(ch.G, dtype=np.uint8), ch.rows, max_batch=2 << 20)
    got = eng3.place_stream(batches)
    for i, (g, res) in enumerate(zip(got, results)):
        assert np.array_equal(g, res), i
    assert np.array_equal(eng3.read_occupancy(), occ)
    st = eng3.stats()
    assert st["placed"] == sum(int(((r["status"] == E.ST_PLACED) & (q["op"] == E.OP_ALLOC)).sum()) for q, r in zip(batches, results))


def test_device_resident_entry_point_matches_host_entry_point():
    import torch
    node_off, occ, rows, req = W.config3(n=70_000)
    eng = make_engine(node_off, occ, rows)
    want = eng.place_batch(req)
    eng.load_inventory(node_off, occ)
    d_in = torch.from_numpy(req.view(np.int64)).cuda()
    d_out = torch.empty_like(d_in)
    torch.cuda.synchronize()
    eng.place_batch_device(len(req), d_in.data_ptr(), d_out.data_ptr())
    eng.synchronize()
    got = d_out.cpu().numpy().view(E.RESULT_DTYPE)
    assert np.array_equal(got, want)
    st = eng.stats()
    assert st["placed"] == int((want["status"] == E.ST_PLACED).sum()) * 2 and st["kernel_launches"] > 0
    # one device-resident chunk: k_small up to 1024 requests, else the chunk path even when it mixes profiles (only a host batch is
    # looked at for that)
    for n, launches in ((700, 1), (5000, 6)):
        eng.load_inventory(node_off, occ)
        want = eng.place_batch(req[:n])
        eng.load_inventory(node_off, occ)
        before = eng.stats()["kernel_launches"]
        eng.place_batch_device(n, d_in.data_ptr(), d_out.data_ptr())
        eng.synchronize()
        assert eng.stats()["kernel_launches"] - before == launches, (n, eng.stats())
        assert np.array_equal(d_out[:n].cpu().numpy().view(E.RESULT_DTYPE), want), n


# ---- partitioned inventory: token ring between engines (the N > 1 device path) on ONE GPU ---------------------------
@pytest.mark.parametrize("n_ranks", [2, 3])
def test_partitioned_ring_on_one_gpu(n_ranks):
    """Several engines in one process, each owning a GPU range, wired with isl_connect_local: the queue-head token of
    every chunk crosses from the last segment of one engine's running kernel to the first segment of the next one's
    (the same mechanism the multi-GPU run uses through CUDA IPC).  Merged results == global sequential first-fit."""
    import torch
    from instaslice_b200 import dist as D
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(4242 + n_ranks)
    G = 4096
    node_off = W.node_offsets(G // 8, 8)
    occ0 = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows)
    ref.load(occ0)
    batches, want, live = [], [], []
    for b in range(6):
        n = 3000 + 500 * b
        req = W.alloc_requests(W.mix_profiles(rng, n))
        for i in range(min(len(live), n // 3)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        res = ref.place(req)
        for r in res[(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)]:
            live.append((int(r["gpu"]), int(r["start"]), int(r["size"])))
        batches.append(req)
        want.append(res)
    sizes = np.array([len(b) for b in batches], dtype=np.uint32)
    d_in = torch.from_numpy(np.concatenate(batches).view(np.int64).copy()).cuda()
    bounds = D.all_bounds(G, n_ranks, align=64)
    engines, outs = [], []
    for r, (lo, hi) in enumerate(bounds):
        eng = make_engine(node_off, occ0, rows)
        eng.set_partition(lo, hi)
        eng.ipc_inbox_handle()                       # allocates the inbox
        engines.append(eng)
        outs.append(torch.empty_like(d_in))
    for r, eng in enumerate(engines):
        eng.connect_local(engines[r + 1] if r + 1 < n_ranks else None, has_prev=r > 0)
    torch.cuda.synchronize()
    for stream_id in (1, 2):                          # twice: the second run re-uses inbox slots with a new stream id
        for eng in engines:
            eng.load_inventory(node_off, occ0)
        for eng, (lo, hi) in zip(engines, bounds):
            eng.set_partition(lo, hi)
        for eng, out in zip(engines, outs):
            eng.place_stream_partitioned(sizes, d_in.data_ptr(), out.data_ptr(), stream_id)
        for eng in engines:
            eng.synchronize()
        merged = np.minimum.reduce([o.cpu().numpy() for o in outs]).view(E.RESULT_DTYPE)
        assert np.array_equal(merged, np.concatenate(want))
        occ = np.concatenate([eng.read_occupancy()[lo:hi] for eng, (lo, hi) in zip(engines, bounds)])
        assert np.array_equal(occ, ref.occupancy())


@pytest.mark.parametrize("n_ranks,window", [(2, 0), (3, 1), (2, 2)])
def test_partitioned_ring_results_gathered_on_the_owner(n_ranks, window):
    """The multi-GPU result path without a collective: every engine behind the owner (rank 0) maps the owner's result array
    (isl_connect_owner_local here, CUDA IPC across processes) and its commit threads store each PLACED record there as well; the
    causal window across ranks counts finished ranks per chunk on the owner (peer atomics).  The owner's array alone == the
    global sequential first-fit."""
    import torch
    from instaslice_b200 import dist as D
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(777 + n_ranks + window)
    G = 4096
    node_off = W.node_offsets(G // 8, 8)
    occ0 = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows)
    ref.load(occ0)
    batches, want, live = [], [], []
    for b in range(7):
        n = 2500 + 400 * b
        req = W.alloc_requests(W.mix_profiles(rng, n))
        for i in range(min(len(live), n // 3)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        res = ref.place(req)
        for r in res[(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)]:
            live.append((int(r["gpu"]), int(r["start"]), int(r["size"])))
        batches.append(req)
        want.append(res)
    sizes = np.array([len(b) for b in batches], dtype=np.uint32)
    total = int(sizes.sum())
    d_in = torch.from_numpy(np.concatenate(batches).view(np.int64).copy()).cuda()
    bounds = D.all_bounds(G, n_ranks, align=64)
    engines = []
    for r, (lo, hi) in enumerate(bounds):
        eng = make_engine(node_off, occ0, rows)
        eng.set_partition(lo, hi)
        eng.ipc_inbox_handle()
        engines.append(eng)
    for r, eng in enumerate(engines):
        eng.connect_local(engines[r + 1] if r + 1 < n_ranks else None, has_prev=r > 0)
        eng.connect_owner_local(engines[0] if r > 0 else None)
        eng.set_ring_world(n_ranks)
        eng.set_causal_window(window)
    torch.cuda.synchronize()
    for stream_id in (11, 12):
        for eng, (lo, hi) in zip(engines, bounds):
            eng.load_inventory(node_off, occ0)
            eng.set_partition(lo, hi)
        for eng in engines:
            eng.place_stream_partitioned(sizes, d_in.data_ptr(), eng.device_results(), stream_id)
        for eng in engines:
            eng.synchronize()
        class _View:            # torch view of the owner's engine-owned result array (no copy)
            __cuda_array_interface__ = {"shape": (total,), "typestr": "<i8", "data": (engines[0].device_results(), False), "version": 3}
        owner = torch.as_tensor(_View(), device="cuda").cpu().numpy().view(E.RESULT_DTYPE)
        assert np.array_equal(owner, np.concatenate(want)), (n_ranks, window, stream_id)
        occ = np.concatenate([eng.read_occupancy()[lo:hi] for eng, (lo, hi) in zip(engines, bounds)])
        assert np.array_equal(occ, ref.occupancy())


# ---- best-fit (extension, SURVEY 8a-ext: no reference counterpart; parity against oracle/ref_fast.cpp best-fit) -----------
def check_best_fit(node_off, occ, rows, batches, quirks=E.QUIRKS_REF_EXACT):
    eng = E.Engine(max_gpus=max(4096, len(occ)), max_batch=1 << 20, quirks=quirks, policy=E.POLICY_BEST_FIT)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    ref = oracle.Fast(node_off, rows, quirks, policy=1)
    ref.load(occ)
    for i, req in enumerate(batches):
        got, want = eng.place_batch(req), ref.place(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (i, bad[:5], got[bad[:5]], want[bad[:5]])
        assert np.array_equal(eng.read_occupancy(), ref.occupancy()), i
    return eng


def test_best_fit_config3():
    node_off, occ, rows, req = W.config3(n=30_000)           # 4096 GPUs: class bitmaps in shared memory
    check_best_fit(node_off, occ, rows, [req])


@pytest.mark.parametrize("G", [37, 4096, 12288])
def test_best_fit_random_with_frees(G):
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(G)
    node_off = np.concatenate([[0], np.cumsum(np.full((G + 7) // 8, 8))]).astype(np.uint32)
    node_off[-1] = G
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows, 0, policy=1)
    ref.load(occ)
    batches, live = [], []
    for b in range(4):
        n = 800 + 400 * b
        req = W.alloc_requests((rng.next(n) % np.uint64(len(rows))).astype(np.uint8))
        for i in range(min(len(live), n // 3)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        res = ref.place(req)
        for r in res[(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)]:
            live.append((int(r["gpu"]), int(r["start"]), int(r["size"])))
        batches.append(req)
    check_best_fit(node_off, occ, rows, batches, quirks=0)


def test_best_fit_prefers_tightest_gpu():
    """Hand-checkable: a 1g request goes to the fullest GPU that still has a free slice, not to the first one."""
    rows = E.make_profiles(tables.A100_40GB)
    eng = E.Engine(max_gpus=4096, max_batch=64, policy=E.POLICY_BEST_FIT)
    eng.load_profiles(rows)
    eng.load_inventory(W.node_offsets(1, 4), np.array([0x00, 0x0F, 0x3F, 0x7F], dtype=np.uint8))
    res = eng.place_batch(W.alloc_requests(np.array([0, 0, 1], dtype=np.uint8)))     # 1g, 1g, 2g
    ref = oracle.Fast(W.node_offsets(1, 4), rows, 3, policy=1)
    ref.load(np.array([0x00, 0x0F, 0x3F, 0x7F], dtype=np.uint8))
    want = ref.place(W.alloc_requests(np.array([0, 0, 1], dtype=np.uint8)))
    assert np.array_equal(res, want)
    assert (int(res["gpu"][0]), int(res["start"][0])) == (2, 6) and (int(res["gpu"][1]), int(res["start"][1])) == (1, 4)


def test_large_inventory_stays_on_the_pipeline():
    """300k GPUs need more pipeline segments than CTAs can be co-resident: every stage then walks several sub-segments per chunk
    (up to 8 x 512 GPUs, 132 stages = 540 672 GPUs per H100); beyond that the engine takes the multi-CTA sweep + single-chain path
    on its own.  Bit-exact either way, also with frees between the batches."""
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(300)
    G = 300_000
    node_off = W.node_offsets(G // 8, 8)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)       # ~75 % busy: long infeasible runs to skip
    batches = [W.alloc_requests(W.mix_profiles(rng, 70_000)), W.alloc_requests(W.mix_profiles(rng, 20_000))]
    ref = oracle.Fast(node_off, rows)
    ref.load(occ)
    want = [ref.place(b) for b in batches]
    eng = make_engine(node_off, occ, rows)
    got = eng.place_stream(batches)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    assert eng.gpu_to_node(G - 1) == G // 8 - 1
    # the pipeline served it: table build + (pre-pass x 2 + ready flag) per fed batch + ONE cooperative launch = 8 (the chunk-by-chunk
    # path needs 6 launches per chunk: 19 for these three chunks)
    assert eng.stats()["kernel_launches"] <= 9
    # a churn stream with frees over the same large inventory, twice (the second run re-uses every buffer)
    live = [(int(r["gpu"]), int(r["start"]), int(r["size"])) for g, b in zip(got, batches) for r in g[g["status"] == E.ST_PLACED]]
    for rep in range(2):
        stream = []
        for n in (30_000, 66_000, 5_000):
            req = W.alloc_requests(W.mix_profiles(rng, n))
            for _ in range(min(len(live), n // 3)):
                g_, s_, z_ = live.pop(int(rng.next1() % len(live)))
                req[int(rng.next1() % n)] = (g_, 0, E.OP_FREE, s_, z_)
            res = ref.place(req)
            live.extend((int(r["gpu"]), int(r["start"]), int(r["size"])) for r in res[(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)])
            stream.append((req, res))
        got2 = eng.place_stream([x[0] for x in stream])
        assert all(np.array_equal(a, b[1]) for a, b in zip(got2, stream)), rep
        assert np.array_equal(eng.read_occupancy(), ref.occupancy()), rep
    # 700k GPUs are beyond 132 x 8 x 512: the single-chain path takes over
    G2 = 700_000
    node_off2 = W.node_offsets(G2 // 8, 8)
    occ2 = ((rng.next(G2) | rng.next(G2)) & np.uint64(0x7F)).astype(np.uint8)
    ref2 = oracle.Fast(node_off2, rows)
    ref2.load(occ2)
    b2 = [W.alloc_requests(W.mix_profiles(rng, 20_000)), W.alloc_requests(W.mix_profiles(rng, 9_000))]
    want2 = [ref2.place(b) for b in b2]
    eng2 = make_engine(node_off2, occ2, rows)
    assert all(np.array_equal(a, b) for a, b in zip(eng2.place_stream(b2), want2))
    assert np.array_equal(eng2.read_occupancy(), ref2.occupancy())


def test_incremental_node_update_vs_python_restatement():
    """SURVEY 8f-1: after Instaslice objects change (the daemonset deletes allocations, dangling slices appear, a pod is
    released), rewriting only the touched nodes' occupancy bytes must leave the engine in the state the reference would compute
    from the mutated custom resources.  The checker is the independent restatement ``ref_py`` run on a deep copy of the SAME
    mutated CRs (occupancy byte per GPU via :306-328, then pod by pod through the node loop :188-232) — not the engine itself."""
    gold = load("regress_crd.json")
    for ci in (5, 2, 7):
        case = gold["cases"][ci % len(gold["cases"])]
        items = copy.deepcopy(case["instaslices"])
        quirks = case["quirks"]
        r = ctl.InstasliceReconciler(items, quirks=quirks)
        pods = [{"uid": p["uid"], "name": p["uid"], "profile": p["profile"]} for p in case["pods"]]
        shadow = copy.deepcopy(items)               # ref_py's world: mutated in lock-step, never touched by the engine mirror
        first = r.place_pending_pods(pods[:6])
        for pod in pods[:6]:
            ref_py.reconcile_gated_pod(shadow, {"uid": pod["uid"], "name": pod["name"]}, pod["profile"], quirks)
        # (1) the daemonset deletes a realised allocation on one node
        victim = next((a for v, a in first if a), None)
        if victim is not None:
            for world in (items, shadow):
                node = next(it for it in world if it["metadata"]["name"] == victim["nodename"])
                node["spec"]["allocations"].pop(victim["podUUID"])
            r.update_node(next(it for it in items if it["metadata"]["name"] == victim["nodename"]))
        # (2) a new dangling slice shows up on another node
        uuid = sorted(items[-1]["spec"]["MigGPUUUID"])[0]
        if ctl.occupancy_byte(items[-1], uuid) & 0x40 == 0:
            for world in (items, shadow):
                world[-1]["spec"].setdefault("prepared", {})["MIG-new"] = {"profile": "1g", "start": 6, "size": 1, "parent": uuid, "podUUID": "", "giinfo": 0, "ciinfo": 0}
            r.update_node(items[-1])
        # (3) a pod is released through the mirror (OR-rebuild of its node)
        second = next((a for v, a in first if a and a is not victim), None)
        if second is not None:
            assert r.release(second["podUUID"])
            next(it for it in shadow if it["metadata"]["name"] == second["nodename"])["spec"]["allocations"].pop(second["podUUID"])
        # engine occupancy == what the reference's rebuild (:306-328) gives on the mutated CRs
        want_occ = [ctl.occupancy_byte(it, u) for it in shadow for u in sorted(it["spec"].get("MigGPUUUID", {}))]
        assert r.engine.read_occupancy().tolist() == want_occ, ci
        # and the remaining pods are placed exactly where ref_py places them on those CRs
        got = r.place_pending_pods(copy.deepcopy(pods[6:]))
        for pod, (verdict, alloc) in zip(pods[6:], got):
            v, placed = ref_py.reconcile_gated_pod(shadow, {"uid": pod["uid"], "name": pod["name"]}, pod["profile"], quirks)
            assert verdict == v, (ci, pod)
            if v == "placed":
                assert (alloc["gpuUUID"], alloc["start"], alloc["size"], alloc["nodename"]) == (placed[0]["gpuUUID"], placed[0]["start"], placed[0]["size"], placed[0]["nodename"])


@pytest.mark.parametrize("quirks", [3, 0])
def test_right_to_left_rows(quirks):
    """SURVEY 8f-4: the reference's RightToLeftPolicy is a stub (:464-469).  The start search honours ROW order (:343-383), so a
    right-to-left policy is the engine fed with reversed rows; the oracle, which walks the rows the same way, is the checker."""
    rows = E.make_profiles(tables.H100_80GB, right_to_left=True)
    assert list(rows[0]["starts"][:7]) == [6, 5, 4, 3, 2, 1, 0]
    rng = W.SplitMix64(5 + quirks)
    G = 3000
    node_off = np.concatenate([[0], np.cumsum(np.full((G + 7) // 8, 8))]).astype(np.uint32)
    node_off[-1] = G
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows, quirks)
    ref.load(occ)
    batches = [W.alloc_requests(W.mix_profiles(rng, n)) for n in (900, 70000, 40)] + [W.alloc_requests(np.zeros(5000, dtype=np.uint8))]   # last: scan mode
    want = [ref.place(b) for b in batches]
    # one empty GPU, one 1g request: lands on slice 6, not 0
    assert oracle.start_for(rows[0], quirks, 0x00) == 6
    for flags in (E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL, 0):
        eng = E.Engine(max_gpus=4096, max_batch=1 << 18, quirks=quirks, flags=flags)
        eng.load_profiles(rows)
        eng.load_inventory(node_off, occ)
        got = eng.place_stream(batches) if flags == 0 else [eng.place_batch(b) for b in batches]
        assert all(np.array_equal(a, b) for a, b in zip(got, want)), flags
        assert np.array_equal(eng.read_occupancy(), ref.occupancy())
