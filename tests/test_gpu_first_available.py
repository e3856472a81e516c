"""Profile alternatives (ISL_FLAG_FIRST_AVAILABLE, include/islplace.h A1-A8) on the H100: k_bestfit's and k_nodefit's pod loops against
the brute force of tests/first_available_fast.cpp, byte for byte (records, final occupancy, stats.placed), through every entry point
that follows A1-A5; A4 and A5 (b) device against device; isl_place_gangs and isl_preempt unchanged by the flag; the codes of A6 and A7;
the reconciler flows in Python and C++.

Return codes on a flagged engine (A6, A7):
  isl_create                          ISL_EINVAL with ISL_FLAG_ALL_NODES, ISL_ERANGE for max_gpus > 2^20, else ISL_OK (any policy)
  isl_place_batch, _range, _device    ISL_OK, pods of alternatives
  isl_place_stream, _device           ISL_OK, one batch after the other
  isl_what_if                         ISL_OK, pods of alternatives
  isl_place_batch_partitioned         ISL_EINVAL
  isl_place_stream_partitioned        ISL_EINVAL
  isl_stream_open                     ISL_EINVAL
  isl_place_gangs, isl_preempt        as without the flag
"""
import copy
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables

import bestfit_fast as BF
import first_available_fast as F
import first_available_oracle as O
import node_score_oracle as NO

pytestmark = pytest.mark.gpu
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG, E.POLICY_MOST_ALLOCATED,
            E.POLICY_LEAST_ALLOCATED]
QUIRKS = [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED]
TABLES3 = [tables.H100_80GB, tables.A30_24GB, tables.A100_40GB]
FA = E.FLAG_FIRST_AVAILABLE


def engine(node_off, rows, occ, policy, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=1 << 16, flags=FA):
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
    occ = np.zeros(G, dtype=np.uint8)
    for x in range(8):
        occ |= ((rng.random(G) < fill).astype(np.uint8) << x)
    return occ


def random_node_off(rng, G, shape):
    if shape == "single":
        return np.arange(G + 1, dtype=np.uint32)
    if shape == "eight":
        return np.concatenate([np.arange(0, G, 8), [G]]).astype(np.uint32)
    sizes = []                                  # "varying": 0 (empty) .. 16 GPUs per node
    while sum(sizes) < G:
        sizes.append(int(rng.choice([0, 1, 2, 4, 7, 8, 8, 8, 16])))
    sizes[-1] -= sum(sizes) - G
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


def random_pods(rng, n, n_names, G, max_run=5, free_share=0.08, handle_base=0):
    """About n requests: pods of 1..max_run alternatives (handle = pod index, some profiles repeated or unknown), FREEs of single busy
    slices and NOOPs between them; two neighbouring pods sometimes share a handle across a FREE or a NOOP."""
    out, pod = [], handle_base
    while len(out) < n:
        r = rng.random()
        if r < free_share:
            out.append((int(rng.integers(0, G)), 0, E.OP_FREE, int(rng.integers(0, 8)), 1))
            continue
        if r < free_share + 0.02:
            out.append((pod, 0, E.OP_NOOP, 0, 0))
            continue
        k = int(rng.integers(1, max_run + 1))
        for _ in range(k):
            p = int(rng.integers(0, n_names)) if rng.random() > 0.03 else E.PROFILE_UNKNOWN
            out.append((pod, p, E.OP_ALLOC, 0, 0))
        if rng.random() > 0.1:                  # else the next pod reuses the handle: one longer run unless something splits it
            pod += 1
    return np.array(out[:n], dtype=E.REQUEST_DTYPE)


def setup(rng, policy, G, n_tables, shape="eight", fill=0.45):
    node_off = random_node_off(rng, G, shape)
    n_nodes = len(node_off) - 1
    if n_tables == 1:
        rows, node_table, n_names = E.make_profiles(tables.H100_80GB), None, len(tables.H100_80GB)
    else:
        names, rows = E.make_profile_tables(TABLES3[:n_tables])
        node_table, n_names = rng.integers(0, n_tables, n_nodes).astype(np.uint8), len(names)
    return node_off, rows, node_table, random_occ(rng, G, fill), n_names


def check(eng, node_off, rows, occ, req, policy, quirks, node_table, lo=0, hi=None, ranged=False):
    """One flagged call against the brute force: records, whole occupancy, stats.placed.  Returns the occupancy after."""
    before = eng.stats()["placed"]
    got = eng.place_batch_range(lo, hi, req) if ranged else eng.place_batch(req)
    want, occ2, placed = F.place(node_off, rows, occ, req, policy, quirks, node_table, lo, hi)
    assert O.as_tuples(got) == O.as_tuples(want)
    assert np.array_equal(eng.read_occupancy(), occ2)
    assert eng.stats()["placed"] - before == placed
    return occ2


@pytest.mark.parametrize("case", O.kat_cases(), ids=lambda c: c["name"])
def test_kat(case):
    node_off, rows, node_table, occ, req, quirks, policy, (lo, hi) = O.case_inputs(case)
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    out = eng.place_batch_range(lo, hi, req) if "range" in case else eng.place_batch(req)
    assert O.as_tuples(out) == O.expected(case)
    assert np.array_equal(eng.read_occupancy(), O.runs(case["occ_after"]))
    eng.close()


@pytest.mark.parametrize("quirks", QUIRKS)
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("n_tables", [1, 3])
def test_random_against_brute_force(policy, quirks, n_tables):
    """Two batches in a row on one engine, then a restricted range and a restricted partition."""
    rng = np.random.default_rng(1000 * policy + 10 * quirks + n_tables)
    G = 1536
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, n_tables, "varying")
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    for _ in range(2):
        occ = check(eng, node_off, rows, occ, random_pods(rng, 3000, n_names, G), policy, quirks, node_table)
    lo, hi = int(node_off[3]) + 1, int(node_off[-4]) - 1             # cuts through nodes
    occ = check(eng, node_off, rows, occ, random_pods(rng, 800, n_names, G), policy, quirks, node_table, lo, hi, ranged=True)
    eng.set_partition(lo, hi)
    check(eng, node_off, rows, occ, random_pods(rng, 800, n_names, G), policy, quirks, node_table, lo, hi)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("G", [4096, 4097])
def test_bestfit_shared_memory_switch(policy, G):
    """k_bestfit keeps its class bitmaps in shared memory up to 4 096 GPUs of one table; k_nodefit's trees live there up to 2 048
    nodes, so single-GPU nodes put node scoring on both sides as well."""
    rng = np.random.default_rng(G + policy)
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 1, "single", fill=0.6)
    eng = engine(node_off, rows, occ, policy)
    check(eng, node_off, rows, occ, random_pods(rng, 2500, n_names, G), policy, E.QUIRKS_REF_EXACT, None)
    eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED])
@pytest.mark.parametrize("nodes", [2048, 2049])
def test_nodefit_shared_memory_switch(policy, nodes):
    rng = np.random.default_rng(nodes + 7 * policy)
    G = 2 * nodes
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 3, "single", fill=0.5)
    node_off = np.arange(0, G + 1, 2, dtype=np.uint32)
    node_table = rng.integers(0, 3, nodes).astype(np.uint8)
    eng = engine(node_off, rows, occ, policy, E.QUIRKS_FIXED, node_table)
    check(eng, node_off, rows, occ, random_pods(rng, 2000, n_names, G), policy, E.QUIRKS_FIXED, node_table)
    eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MOST_ALLOCATED])
def test_inventory_at_the_cap(policy):
    """2^20 GPUs, the largest inventory a flagged engine takes (A7), nearly full so that pods fall back."""
    rng = np.random.default_rng(20 + policy)
    G = 1 << 20
    node_off = np.concatenate([np.arange(0, G, 8), [G]]).astype(np.uint32)
    occ = random_occ(rng, G, 0.9)
    rows = E.make_profiles(tables.H100_80GB)
    eng = engine(node_off, rows, occ, policy)
    check(eng, node_off, rows, occ, random_pods(rng, 150, len(rows), G, free_share=0.0), policy, E.QUIRKS_REF_EXACT, None)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_runs_across_block_edges(policy):
    """Runs that straddle the 32-request blocks of the kernels' loops: runs of 24, 16, 40 (repeated profiles) and 33; pods of one up to
    request 30, a NOOP at 31 carrying the handle of the pod that opens the next block, which is therefore a pod of its own."""
    rng = np.random.default_rng(policy + 77)
    G = 512
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 1, fill=0.7)
    groups = [[int(rng.integers(0, n_names)) for _ in range(24)], [int(rng.integers(0, n_names)) for _ in range(16)],
              [5, 5, 4, 4, 3, 3, 2, 2, 1, 1, 0, 0] * 3 + [0, 0, 0, 0], [int(rng.integers(0, n_names)) for _ in range(33)]]
    req = F.pods(groups)
    pad = (31 - len(req)) % 32
    ones = F.pods([[int(rng.integers(0, n_names))] for _ in range(pad)], list(range(10, 10 + pad)))
    noop = np.array([(99, 0, E.OP_NOOP, 0, 0)], dtype=E.REQUEST_DTYPE)
    tail = F.pods([[5, 4, 3, 2, 1, 0] * 7], [99])
    req = np.concatenate([req, ones, noop, tail])
    assert len(req) - len(tail) == 32 * ((len(req) - len(tail)) // 32)
    eng = engine(node_off, rows, occ, policy)
    check(eng, node_off, rows, occ, req, policy, E.QUIRKS_REF_EXACT, None)
    eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_stream_batches_cut_runs(policy):
    """isl_place_stream: each batch is its own (A1), so a batch edge inside a would-be run makes two pods; the device stream equals the
    brute force batch after batch."""
    rng = np.random.default_rng(policy + 5)
    G = 1024
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 3)
    req = random_pods(rng, 3000, n_names, G)
    sizes = [700, 1, 33, 1266, 1000]
    assert sum(sizes) == len(req)
    batches = np.split(req, np.cumsum(sizes)[:-1])
    eng = engine(node_off, rows, occ, policy, E.QUIRKS_FIXED, node_table)
    got = eng.place_stream(batches)
    for b, batch in enumerate(batches):
        want, occ, _ = F.place(node_off, rows, occ, batch, policy, E.QUIRKS_FIXED, node_table)
        assert O.as_tuples(got[b]) == O.as_tuples(want), b
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_MIN_FRAG, E.POLICY_LEAST_ALLOCATED])
def test_device_batch_and_what_if(policy):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(policy + 11)
    G = 1024
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 1)
    eng = engine(node_off, rows, occ, policy)
    plan = random_pods(rng, 1500, n_names, G)
    out, before, after = eng.what_if(plan)
    want, _, _ = F.place(node_off, rows, occ, plan, policy)
    assert O.as_tuples(out) == O.as_tuples(want)
    assert np.array_equal(eng.read_occupancy(), occ)                    # the live state is put back
    d_in = torch.from_numpy(plan.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(plan) * 8, dtype=torch.uint8, device="cuda")
    eng.place_batch_device(len(plan), d_in.data_ptr(), d_out.data_ptr())
    eng.synchronize()
    got = d_out.cpu().numpy().view(E.RESULT_DTYPE)
    assert O.as_tuples(got) == O.as_tuples(want)
    eng.close()


@pytest.mark.parametrize("quirks", QUIRKS)
@pytest.mark.parametrize("policy", POLICIES)
def test_a4_pods_of_one_equal_unflagged(policy, quirks):
    """A4 device against device: distinct handles, so a flagged call equals the unflagged engine's (for first-fit the small kernel and
    the segment pipeline), records, occupancy and stats.placed; on a partition as well."""
    rng = np.random.default_rng(policy * 3 + quirks)
    G = 2048
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 3)
    req = random_pods(rng, 6000, n_names, G, max_run=1)
    req["handle"][req["op"] == E.OP_ALLOC] = np.arange(int((req["op"] == E.OP_ALLOC).sum()))
    for part in [None, (int(node_off[5]) + 3, G - 100)]:
        engs = [engine(node_off, rows, occ, policy, quirks, node_table, flags=f) for f in (FA, 0)]
        res = []
        for eng in engs:
            if part:
                eng.set_partition(*part)
            res.append((eng.place_batch(req), eng.place_batch(req[:700]), eng.read_occupancy(), eng.stats()["placed"]))
        (a, a2, oa, pa), (b, b2, ob, pb) = res
        assert np.array_equal(a, b) and np.array_equal(a2, b2) and np.array_equal(oa, ob) and pa == pb
        for eng in engs:
            eng.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_a5b_chosen_only_equals_unflagged(policy):
    """A5 (b): each pod's chosen alternative alone, every other alternative a NOOP, on the unflagged engine: same PLACED records, same
    occupancy."""
    rng = np.random.default_rng(policy + 500)
    G = 1024
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 1, fill=0.55)
    req = random_pods(rng, 4000, n_names, G)
    flagged = engine(node_off, rows, occ, policy)
    plain = engine(node_off, rows, occ, policy, flags=0)
    got = flagged.place_batch(req)
    alone = plain.place_batch(O.chosen_only(req, got))
    placed = got["status"] == E.ST_PLACED
    assert np.array_equal(alone["status"] == E.ST_PLACED, placed)
    assert np.array_equal(alone[placed], got[placed])
    assert np.array_equal(flagged.read_occupancy(), plain.read_occupancy())
    flagged.close(); plain.close()


@pytest.mark.parametrize("policy", POLICIES)
def test_gangs_and_preempt_ignore_the_flag(policy):
    """isl_place_gangs and isl_preempt answer the same on flagged and unflagged engines (handles stay opaque in gangs)."""
    from test_gpu_preempt import random_requests, random_state
    rng = np.random.default_rng(policy + 900)
    G = 1024
    node_off = np.concatenate([np.arange(0, G, 8), [G]]).astype(np.uint32)
    rows = E.make_profiles(tables.H100_80GB)
    occ = random_occ(rng, G, 0.5)
    req = random_pods(rng, 600, len(rows), G, free_share=0.0)
    gang_off = np.unique(np.concatenate([[0], np.sort(rng.integers(1, len(req), 150)), [len(req)]])).astype(np.uint32)
    refusals = (policy in (E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED))     # node scoring without ISL_FLAG_GANG_NODE_SCORE
    out = []
    for f in (FA, 0):
        eng = engine(node_off, rows, occ, policy, flags=f)
        if refusals:
            with pytest.raises(E.EngineError) as ei:
                eng.place_gangs(req, gang_off)
            g = ei.value.code
        else:
            g = eng.place_gangs(req, gang_off)
        occ_g = eng.read_occupancy()
        pocc, vic = random_state(np.random.default_rng(policy), G, 1, len(rows), 0.97)
        eng.load_inventory(node_off, pocc)
        preq, prio = random_requests(np.random.default_rng(policy + 1), 256, len(rows))
        res, evict = eng.preempt(preq, prio, vic)
        out.append((g, occ_g, res, evict))
        eng.close()
    (g1, o1, r1, e1), (g2, o2, r2, e2) = out
    assert (g1 == g2) if refusals else np.array_equal(g1, g2)
    assert np.array_equal(o1, o2) and np.array_equal(r1, r2) and np.array_equal(e1, e2)
    if not refusals:
        want, _ = BF.place_gangs(node_off, rows, occ, req, gang_off, policy=policy)
        assert np.array_equal(g1, want)


@pytest.mark.parametrize("policy", POLICIES)
def test_codes_and_refusals_change_nothing(policy):
    lib = E.load_library()
    for flags, max_gpus, rc in [(FA | E.FLAG_ALL_NODES, 4096, E.EINVAL), (FA, (1 << 20) + 1, E.ERANGE), (FA, 1 << 20, E.OK),
                                (FA | E.FLAG_GANG_PREEMPT, 4096, E.OK)]:
        h = C.c_void_p()
        cfg = E.Config(E.ABI_VERSION, policy, E.QUIRKS_REF_EXACT, -1, max_gpus, 1024, flags, 0)
        assert lib.isl_create(C.byref(cfg), C.byref(h)) == rc
        assert bool(h.value) == (rc == E.OK)
        if h.value:
            lib.isl_destroy(h)
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(policy + 3)
    G = 1024
    node_off, rows, node_table, occ, n_names = setup(rng, policy, G, 1)
    eng = engine(node_off, rows, occ, policy)
    req = random_pods(rng, 256, n_names, G)
    d_in = torch.from_numpy(req.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(req) * 8, dtype=torch.uint8, device="cuda")
    heads = torch.zeros(E.MAX_PROFILES * 4, dtype=torch.int32, device="cuda")
    sizes = np.array([len(req)], dtype=np.uint32)
    h = eng._h
    assert lib.isl_place_batch_partitioned(h, len(req), d_in.data_ptr(), d_out.data_ptr(), None, heads.data_ptr()) == E.EINVAL
    assert lib.isl_place_stream_partitioned(h, 1, sizes.ctypes.data_as(C.c_void_p), d_in.data_ptr(), d_out.data_ptr(), 7) == E.EINVAL
    assert lib.isl_stream_open(h, 1) == E.EINVAL
    assert np.array_equal(eng.read_occupancy(), occ)
    check(eng, node_off, rows, occ, req, policy, E.QUIRKS_REF_EXACT, None)      # still works, no stream was left open
    eng.close()


def _items(rng, G):
    node_off = random_node_off(rng, G, "varying")
    node_table = rng.integers(0, 2, len(node_off) - 1).astype(np.uint8)
    occ = random_occ(rng, G, 0.55)
    return node_off, node_table, occ, NO.items_from(node_off, occ, ["h100-80gb", "a30-24gb"], node_table)


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_LEAST_ALLOCATED])
def test_reconciler_fallbacks(policy):
    """place_pending_pods on a first_available reconciler: the chosen profile is the first of the pod's names the brute force places,
    and its AllocationDetails carry that profile's size and GI / CI ids; an unflagged reconciler refuses fallbacks."""
    rng = np.random.default_rng(policy + 31)
    node_off, node_table, occ, items = _items(rng, 200)
    names = [r[0] for r in tables.H100_80GB] + [r[0] for r in tables.A30_24GB]
    pods = []
    for i in range(300):
        alts = [names[int(k)] for k in rng.integers(0, len(names), int(rng.integers(1, 4)))]
        pods.append({"uid": "pod-%d" % i, "name": "pod-%d" % i, "namespace": "default", "profile": alts[0], "fallbacks": alts[1:]})
    r = ctl.InstasliceReconciler(copy.deepcopy(items), policy=policy, first_available=True)
    flat = [n for p in pods for n in [p["profile"], *p["fallbacks"]]]
    req = r._requests(flat, [i for i, p in enumerate(pods) for _ in [p["profile"], *p["fallbacks"]]])
    want, _, _ = F.place(r.node_off, r.rows, r.engine.read_occupancy(), req, policy, E.QUIRKS_REF_EXACT, np.array(r.node_table, np.uint8))
    got = r.place_pending_pods(pods)
    gpu_names = [u for it in items for u in sorted(it["spec"]["MigGPUUUID"])]
    k = 0
    for pod, (verdict, alloc) in zip(pods, got):
        alts = [pod["profile"], *pod["fallbacks"]]
        recs = want[k:k + len(alts)]
        k += len(alts)
        hit = [a for a, w in zip(alts, recs) if w["status"] == E.ST_PLACED]
        if not hit:
            assert verdict == "none"
            continue
        w = recs[alts.index(hit[0])]
        assert verdict == "placed" and alloc["profile"] == hit[0]
        assert (alloc["gpuUUID"], alloc["start"]) == (gpu_names[int(w["gpu"])], int(w["start"]))
        node = r.items[r.node_of_uuid[alloc["gpuUUID"]]]
        size, gi, ci, cieng = r.extractGpuProfile(node, hit[0])
        assert (alloc["size"], alloc["giprofileid"], alloc["ciProfileid"], alloc["ciengprofileid"]) == (size, gi, ci, cieng)
        assert node["spec"]["allocations"][pod["uid"]] is alloc
    plain = ctl.InstasliceReconciler(copy.deepcopy(items), policy=policy)
    with pytest.raises(ValueError):
        plain.place_pending_pods(pods)
    # pods without fallbacks: a flagged reconciler answers exactly as an unflagged one
    bare = [{k: v for k, v in p.items() if k != "fallbacks"} for p in pods]
    a = ctl.InstasliceReconciler(copy.deepcopy(items), policy=policy, first_available=True).place_pending_pods(bare)
    b = ctl.InstasliceReconciler(copy.deepcopy(items), policy=policy).place_pending_pods(bare)
    assert a == b


def test_reconciler_fallbacks_with_orphans():
    """With a dangling Prepared slice (the veto can fire) every pod is one engine call with its whole run: the same answers as one call."""
    rng = np.random.default_rng(8)
    node_off, node_table, occ, items = _items(rng, 64)
    for it in items:
        if it["spec"]["MigGPUUUID"]:
            it["spec"]["prepared"]["orphan"] = {"parent": sorted(it["spec"]["MigGPUUUID"])[0], "start": 7, "size": 1, "podUUID": "gone"}
            break
    pods = [{"uid": "p%d" % i, "name": "p%d" % i, "profile": "7g.80gb", "fallbacks": ["4g.40gb", "1g.10gb"]} for i in range(40)]
    one_call = ctl.InstasliceReconciler(copy.deepcopy(items), first_available=True)
    one_call._has_orphans = False                   # the same pods in one engine call, for comparison
    want = one_call.place_pending_pods(copy.deepcopy(pods))
    r = ctl.InstasliceReconciler(items, first_available=True)
    assert r._has_orphans
    got = r.place_pending_pods(pods)
    assert [v for v, _ in got] == [v for v, _ in want]
    assert [(a["profile"], a["gpuUUID"], a["start"]) for _, a in got if a] == [(a["profile"], a["gpuUUID"], a["start"]) for _, a in want if a]


def test_host_mirror_first_available_selftest(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_first_available_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(root, "tests", "host_mirror_first_available_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr

