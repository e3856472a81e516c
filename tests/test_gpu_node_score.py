"""Node scoring (ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED) on the H100: k_nodefit against the brute force of
tests/node_score_fast.cpp, records and final occupancy byte-identical, through every entry point that accepts the policies; the
hand-worked vectors; every refusal; isl_preempt on such an engine; the reconciler flows in Python and C++.

Return codes of the new policies per entry point (include/islplace.h, node scoring rules 6 and 7):
  isl_create                         ISL_EINVAL with ISL_FLAG_ALL_NODES, ISL_ERANGE for max_gpus > 2^20, else ISL_OK
  isl_place_batch, _range, _device   ISL_OK
  isl_place_stream, _device          ISL_OK
  isl_what_if, isl_capacity          ISL_OK
  isl_free_batch, isl_eval_starts    ISL_OK
  isl_set_partition, node tables     ISL_OK
  isl_preempt                        ISL_OK, scan order ascending canonical
  isl_place_batch_partitioned        ISL_EINVAL
  isl_place_stream_partitioned       ISL_EINVAL
  isl_stream_open                    ISL_EINVAL
  isl_place_gangs                    ISL_EINVAL
"""
import copy
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import node_offsets

import node_score_fast as NF
import node_score_oracle as NO
import preempt_fast as PF

pytestmark = pytest.mark.gpu
POLICIES = [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED]
TABLES3 = [tables.H100_80GB, tables.A30_24GB, tables.A100_40GB]


def engine(node_off, rows, occ, policy, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=0):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if rows.ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


def random_occ(rng, G, fill):
    """Occupancy of random spans; about `fill` of the slices busy."""
    occ = np.zeros(G, dtype=np.uint8)
    for x in range(8):
        occ |= ((rng.random(G) < fill).astype(np.uint8) << x)
    return occ


def random_batch(rng, n, n_names, G, occ, free_share=0.1):
    """ALLOCs of random profiles, some FREEs of busy single slices, a few unknown profiles and NOOPs."""
    req = np.zeros(n, dtype=E.REQUEST_DTYPE)
    req["handle"] = np.arange(n)
    req["profile"] = rng.integers(0, n_names, n)
    req["op"] = E.OP_ALLOC
    kind = rng.random(n)
    frees = np.flatnonzero(kind < free_share)
    g = rng.integers(0, G, len(frees))
    req["handle"][frees] = g
    req["op"][frees] = E.OP_FREE
    req["start"][frees] = rng.integers(0, 8, len(frees))
    req["size"][frees] = 1
    odd = (kind >= free_share) & (kind < free_share + 0.02)
    req["profile"][odd] = E.PROFILE_UNKNOWN
    req["op"][(kind >= free_share + 0.02) & (kind < free_share + 0.03)] = E.OP_NOOP
    return req


def random_node_off(rng, G, shape):
    if shape == "single":
        return np.arange(G + 1, dtype=np.uint32)
    if shape == "eight":
        return node_offsets(G // 8, 8) if G >= 8 else np.array([0, G], dtype=np.uint32)
    sizes = []                                  # "varying": 0 (empty) .. 16 GPUs per node
    while sum(sizes) < G:
        sizes.append(int(rng.choice([0, 1, 2, 4, 7, 8, 8, 8, 16])))
    sizes[-1] -= sum(sizes) - G
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


@pytest.mark.parametrize("case", NO.kat_cases(), ids=lambda c: c["name"])
def test_kat(case):
    node_off, rows, node_table, occ, req, quirks, policy, (lo, hi) = NO.case_inputs(case)
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    out = eng.place_batch_range(lo, hi, req) if "range" in case else eng.place_batch(req)
    assert [tuple(int(x) for x in r) for r in out] == NO.expected(case)
    assert np.array_equal(eng.read_occupancy(), NO.runs(case["occ_after"]))
    eng.close()


CASES = [  # G, node shape, n_tables, requests; 2048 / 2049 single-GPU nodes straddle the shared-memory tree limit
    (1, "single", 1, 64),
    (7, "varying", 2, 300),
    (4096, "eight", 1, 5000),
    (2048, "single", 1, 3000),
    (2049, "single", 2, 3000),
    (65536, "single", 1, 4000),
    (65536, "varying", 3, 4000),
    (1 << 20, "eight", 1, 300),
]


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("G,shape,n_tables,n", CASES)
def test_random_against_checker(G, shape, n_tables, n, policy, quirks):
    rng = np.random.default_rng(G + n_tables * 7 + policy * 3 + quirks)
    node_off = random_node_off(rng, G, shape)
    names, rows = E.make_profile_tables(TABLES3[:n_tables])
    node_table = rng.integers(0, n_tables, len(node_off) - 1).astype(np.uint8) if n_tables > 1 else None
    occ = random_occ(rng, G, 0.55)
    req = random_batch(rng, n, len(names), G, occ)
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    got = eng.place_batch(req)
    want, after = NF.place(node_off, rows, occ, req, policy, quirks, node_table)
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (bad[:5], got[bad[:5]], want[bad[:5]])
    assert (got["status"] == E.ST_PLACED).any()
    assert np.array_equal(eng.read_occupancy(), after)
    st = eng.stats()
    assert st["placed"] == int((got["status"] == E.ST_PLACED).sum())
    eng.close()


def _setup(policy, G=4096, n_tables=2, seed=3):
    rng = np.random.default_rng(seed + policy)
    node_off = random_node_off(rng, G, "varying")
    names, rows = E.make_profile_tables(TABLES3[:n_tables])
    node_table = rng.integers(0, n_tables, len(node_off) - 1).astype(np.uint8)
    occ = random_occ(rng, G, 0.5)
    return rng, node_off, names, rows, node_table, occ


@pytest.mark.parametrize("policy", POLICIES)
def test_range_cutting_nodes_and_partition(policy):
    rng, node_off, names, rows, node_table, occ = _setup(policy)
    lo, hi = int(node_off[3]) + 1, int(node_off[-4]) - 1         # both bounds inside a node (nodes of >= 2 GPUs are common)
    req = random_batch(rng, 2000, len(names), len(occ), occ)
    eng = engine(node_off, rows, occ, policy, node_table=node_table)
    got = eng.place_batch_range(lo, hi, req)
    want, after = NF.place(node_off, rows, occ, req, policy, node_table=node_table, lo=lo, hi=hi)
    assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), after)
    eng.set_partition(lo, hi)                                     # the same range as the engine's partition
    req2 = random_batch(rng, 2000, len(names), len(occ), after)
    got = eng.place_batch(req2)
    want, after2 = NF.place(node_off, rows, after, req2, policy, node_table=node_table, lo=lo, hi=hi)
    assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), after2)
    cap = eng.capacity()                                          # policy-independent, inside the partition
    ff = engine(node_off, rows, after2, E.POLICY_FIRST_FIT, node_table=node_table)
    ff.set_partition(lo, hi)
    assert np.array_equal(cap, ff.capacity())
    ff.close()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_device_stream_and_what_if(policy):
    torch = pytest.importorskip("torch")
    rng, node_off, names, rows, node_table, occ = _setup(policy, G=8192, n_tables=1, seed=11)
    eng = engine(node_off, rows, occ, policy)
    ref_occ = occ.copy()
    # isl_place_batch_device
    req = random_batch(rng, 3000, len(names), len(occ), occ)
    d_in = torch.from_numpy(req.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(req) * 8, dtype=torch.uint8, device="cuda")
    eng.place_batch_device(len(req), d_in.data_ptr(), d_out.data_ptr())
    eng.synchronize()
    want, ref_occ = NF.place(node_off, rows, ref_occ, req, policy)
    assert np.array_equal(d_out.cpu().numpy().view(E.RESULT_DTYPE), want)
    # isl_place_stream, pageable buffers, several batches: one isl_place_batch each, in order
    batches = [random_batch(rng, k, len(names), len(occ), ref_occ) for k in (1, 700, 0, 5000, 33)]
    got = eng.place_stream(batches)
    for b, g in zip(batches, got):
        want, ref_occ = NF.place(node_off, rows, ref_occ, b, policy)
        assert np.array_equal(g, want)
    assert np.array_equal(eng.read_occupancy(), ref_occ)
    # isl_place_stream from pinned buffers
    batches = [random_batch(rng, k, len(names), len(occ), ref_occ) for k in (4000, 17, 2500)]
    sizes = np.array([len(b) for b in batches], dtype=np.uint32)
    h_in, h_out = E.PinnedArray(int(sizes.sum()), E.REQUEST_DTYPE), E.PinnedArray(int(sizes.sum()), E.RESULT_DTYPE)
    h_in.array[:] = np.concatenate(batches)
    eng.place_stream_ptr(sizes, h_in.ptr, h_out.ptr, device=False)
    off = 0
    for b in batches:
        want, ref_occ = NF.place(node_off, rows, ref_occ, b, policy)
        assert np.array_equal(h_out.array[off:off + len(b)], want)
        off += len(b)
    h_in.free(); h_out.free()
    # isl_place_stream_device
    b = random_batch(rng, 1500, len(names), len(occ), ref_occ)
    d_in = torch.from_numpy(np.concatenate([b, b]).view(np.uint8).copy()).cuda()
    d_out = torch.zeros(2 * len(b) * 8, dtype=torch.uint8, device="cuda")
    eng.place_stream_ptr(np.array([len(b), len(b)], dtype=np.uint32), d_in.data_ptr(), d_out.data_ptr(), device=True)
    eng.synchronize()
    for k in range(2):
        want, ref_occ = NF.place(node_off, rows, ref_occ, b, policy)
        assert np.array_equal(d_out.cpu().numpy().view(E.RESULT_DTYPE)[k * len(b):(k + 1) * len(b)], want)
    assert np.array_equal(eng.read_occupancy(), ref_occ)
    # isl_what_if: the answer of the plan, the live state restored
    plan = random_batch(rng, 2000, len(names), len(occ), ref_occ)
    got, _before, _after = eng.what_if(plan)
    want, _ = NF.place(node_off, rows, ref_occ, plan, policy)
    assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), ref_occ)
    # isl_free_batch, isl_eval_starts
    busy = np.flatnonzero(ref_occ & 1)[:50]
    spans = np.zeros(len(busy), dtype=E.SPAN_DTYPE)
    spans["gpu"], spans["start"], spans["size"] = busy, 0, 1
    eng.free_batch(spans)
    ref_occ[busy] &= 0xFE
    assert np.array_equal(eng.read_occupancy(), ref_occ)
    assert eng.eval_starts(0, np.arange(256, dtype=np.uint8))[0] == 0
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_empty_partition(policy):
    rng, node_off, names, rows, node_table, occ = _setup(policy, G=512, n_tables=1)
    eng = engine(node_off, rows, occ, policy)
    eng.set_partition(100, 100)
    req = random_batch(rng, 500, len(names), len(occ), occ, free_share=0.3)
    got = eng.place_batch(req)
    want, after = NF.place(node_off, rows, occ, req, policy, lo=100, hi=100)
    assert np.array_equal(got, want) and np.array_equal(after, occ)
    assert np.array_equal(eng.read_occupancy(), occ)
    assert not (got["status"] == E.ST_PLACED).any()
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_refusals_change_nothing(policy):
    lib = E.load_library()
    import ctypes as C
    for flags, max_gpus, rc in [(E.FLAG_ALL_NODES, 4096, E.EINVAL), (0, (1 << 20) + 1, E.ERANGE)]:
        h = C.c_void_p()
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, max_gpus, 1024, flags, 0)
        assert lib.isl_create(C.byref(cfg), C.byref(h)) == rc and not h.value
    torch = pytest.importorskip("torch")
    rng, node_off, names, rows, node_table, occ = _setup(policy, G=1024, n_tables=1)
    eng = engine(node_off, rows, occ, policy)
    req = random_batch(rng, 64, len(names), len(occ), occ)
    d_in = torch.from_numpy(req.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(req) * 8, dtype=torch.uint8, device="cuda")
    heads = torch.zeros(E.MAX_PROFILES * 4, dtype=torch.int32, device="cuda")
    sizes = np.array([len(req)], dtype=np.uint32)
    h = eng._h
    assert lib.isl_place_batch_partitioned(h, len(req), d_in.data_ptr(), d_out.data_ptr(), None, heads.data_ptr()) == E.EINVAL
    assert lib.isl_place_stream_partitioned(h, 1, sizes.ctypes.data_as(C.c_void_p), d_in.data_ptr(), d_out.data_ptr(), 7) == E.EINVAL
    assert lib.isl_stream_open(h, 4) == E.EINVAL
    gang_off = np.array([0, 2, len(req)], dtype=np.uint32)
    out = np.zeros(len(req), dtype=E.RESULT_DTYPE)
    assert lib.isl_place_gangs(h, 2, gang_off.ctypes.data_as(C.c_void_p), req.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)) == E.EINVAL
    assert np.array_equal(eng.read_occupancy(), occ)
    got = eng.place_batch(req)                                    # the engine still works, no stream was left open
    want, _ = NF.place(node_off, rows, occ, req, policy)
    assert np.array_equal(got, want)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_preempt_scans_ascending(policy):
    """isl_preempt on a node-scoring engine: k_preempt with the ascending canonical scan order of rule 5."""
    from test_gpu_preempt import random_requests, random_state
    rng = np.random.default_rng(policy)
    G = 4096
    node_off = node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ, vic = random_state(rng, G, 1, len(rows), 0.97)
    req, prio = random_requests(rng, 256, len(rows))
    eng = engine(node_off, rows, occ, policy)
    out, evict = eng.preempt(req, prio, vic)
    rc, want, want_ev = PF.preempt(node_off, rows, occ, req, prio, vic, policy=E.POLICY_FIRST_FIT)
    assert rc == E.OK and np.array_equal(out, want) and np.array_equal(evict, want_ev)
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_reconciler_commits_into_the_crs(policy):
    """The Python reconciler on a node-scoring engine: every PLACED pod becomes an Allocations entry of the node the brute force chose."""
    rng = np.random.default_rng(policy + 40)
    node_off = random_node_off(rng, 300, "varying")
    node_table = rng.integers(0, 2, len(node_off) - 1).astype(np.uint8)
    occ = random_occ(rng, 300, 0.4)
    items = NO.items_from(node_off, occ, ["h100-80gb", "a30-24gb"], node_table)
    names = [r[0] for r in tables.H100_80GB] + [r[0] for r in tables.A30_24GB]
    pods = [{"uid": "pod-%d" % i, "name": "pod-%d" % i, "namespace": "default", "profile": names[int(rng.integers(0, len(names)))]}
            for i in range(400)]
    want = NO.place_cr(copy.deepcopy(items), [{"op": "alloc", "profile": p["profile"], "uid": p["uid"]} for p in pods], policy)
    r = ctl.InstasliceReconciler(items, policy=policy)
    assert r.engine is not None
    got = r.place_pending_pods(pods)
    gpu_names = [u for it in items for u in sorted(it["spec"]["MigGPUUUID"])]
    for pod, (verdict, alloc), w in zip(pods, got, want):
        if w[3] != E.ST_PLACED:
            assert verdict == "none"
            continue
        assert verdict == "placed", pod
        assert (alloc["gpuUUID"], int(alloc["start"]), int(alloc["size"])) == (gpu_names[w[0]], w[1], w[2])
        node = items[int(np.searchsorted(node_off, w[0], side="right")) - 1]
        assert node["spec"]["allocations"][pod["uid"]]["gpuUUID"] == gpu_names[w[0]]


def test_host_mirror_node_score_selftest(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_node_score_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(root, "tests", "host_mirror_node_score_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
