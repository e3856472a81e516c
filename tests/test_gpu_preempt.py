"""Priority preemption (isl_preempt) on the H100: k_victim_map + k_preempt against the brute-force restatement of tests/preempt_fast.cpp,
records and evict rows byte-identical; the known answers; the query leaves every piece of engine state as it found it; every error code
of rules 2, 3 and 6; and the preempt -> release -> place flow through the controller."""
import random

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import node_offsets

import preempt_fast as PF
import preempt_oracle as PO
from test_preempt_oracle import random_cluster, random_pods

pytestmark = pytest.mark.gpu
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, max_batch=4096, flags=0):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if rows.ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    return eng


@pytest.mark.parametrize("case", PO.kat_cases(), ids=lambda c: c["name"])
def test_kat(case):
    node_off, rows, node_table, occ, req, prio, vic, quirks, policy = PO.case_inputs(case)
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    out, evict = eng.preempt(req, prio, vic)
    recs, ev = PO.expected(case)
    assert [tuple(int(x) for x in r) for r in out] == recs
    assert [[int(k) for k in row if k != E.GPU_NONE] for row in evict] == ev
    assert (evict[[r[3] != E.ST_PLACED for r in recs]] == E.GPU_NONE).all()
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()


def random_state(rng, G, n_tables, n_names, busy_share=0.93):
    """Occupancy built from random spans, a span busy with probability busy_share; about 70 % of the busy spans are listed as victims with random priorities (some 255), the rest
    stay pinned.  Vectorised per slot position so that 65 536 GPUs take well under a second."""
    occ = np.zeros(G, dtype=np.uint8)
    vic = []
    pos = np.zeros(G, dtype=np.int64)
    while True:
        live = np.flatnonzero(pos < 8)
        if len(live) == 0:
            break
        size = np.minimum(rng.integers(1, 5, len(live)), 8 - pos[live])
        kind = rng.random(len(live))
        busy = kind < busy_share
        g, s, z = live[busy], pos[live][busy], size[busy]
        occ[g] |= (((1 << z) - 1) << s).astype(np.uint8)
        listed = rng.random(len(g)) < 0.7
        pr = np.where(rng.random(len(g)) < 0.05, 255, rng.integers(0, 8, len(g)))
        for a, b, c, d in zip(g[listed], s[listed], z[listed], pr[listed]):
            vic.append((a, b, c, d, 0))
        pos[live] += size
    vic = np.array(vic, dtype=E.VICTIM_DTYPE)
    return occ, vic[rng.permutation(len(vic))]


def random_requests(rng, n, n_names):
    req = np.zeros(n, dtype=E.REQUEST_DTYPE)
    req["handle"] = np.arange(n)
    req["profile"] = rng.integers(0, n_names, n)
    req["op"] = E.OP_ALLOC
    odd = rng.random(n) < 0.03                       # unknown profiles and NOOPs are answered in place
    req["profile"][odd & (rng.random(n) < 0.5)] = E.PROFILE_UNKNOWN
    req["op"][odd & (req["profile"] != E.PROFILE_UNKNOWN)] = E.OP_NOOP
    return req, rng.integers(1, 10, n).astype(np.uint8)


CASES = [  # G, policy, quirks, node tables, preemptors
    (1, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT, 1, 64),
    (7, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_FIXED, 2, 64),
    (7, E.POLICY_MIN_FRAG, E.QUIRKS_REF_EXACT, 1, 1),
    (4096, E.POLICY_BEST_FIT, E.QUIRKS_REF_EXACT, 2, 1024),
    (4096, E.POLICY_FIRST_FIT, E.QUIRKS_FIXED, 3, 64),
    (4096, E.POLICY_MIN_FRAG, E.QUIRKS_FIXED, 1, 1),
    (65536, E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT, 1, 1024),
    (65536, E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT, 2, 64),
    (65536, E.POLICY_BEST_FIT, E.QUIRKS_FIXED, 3, 1),
]


@pytest.mark.parametrize("G,policy,quirks,n_tables,n", CASES)
def test_random_against_checker(G, policy, quirks, n_tables, n):
    rng = np.random.default_rng(G * 31 + policy * 7 + quirks + n)
    node_off = node_offsets(max(1, G // 8), 8) if G >= 8 else np.array([0, G], dtype=np.uint32)
    names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB][:n_tables])
    node_table = (rng.integers(0, n_tables, len(node_off) - 1)).astype(np.uint8) if n_tables > 1 else None
    occ, vic = random_state(rng, G, n_tables, len(names), 1 - min(0.07, 64 / G))      # nearly full: most pods need an eviction
    req, prio = random_requests(rng, n, len(names))
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    out, evict = eng.preempt(req, prio, vic)
    rc, want, want_ev = PF.preempt(node_off, rows, occ, req, prio, vic, quirks, policy, node_table)
    assert rc == E.OK
    bad = np.flatnonzero(out != want)
    assert len(bad) == 0, (bad[:5], out[bad[:5]], want[bad[:5]])
    assert np.array_equal(evict, want_ev)
    assert (out["status"] == E.ST_PLACED).any() and (evict != E.GPU_NONE).any() or n == 1
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
@pytest.mark.parametrize("lo,hi", [(3, 4098), (1001, 1002), (0, 65531)])
def test_partition(policy, lo, hi):
    """Inside isl_set_partition at unaligned bounds: only the range is searched, victims outside it are ignored."""
    rng = np.random.default_rng(lo + hi + policy)
    G = 65536
    node_off = node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ, vic = random_state(rng, G, 1, len(rows))
    req, prio = random_requests(rng, 64, len(rows))
    eng = engine(node_off, rows, occ, policy)
    eng.set_partition(lo, hi)
    out, evict = eng.preempt(req, prio, vic)
    _rc, want, want_ev = PF.preempt(node_off, rows, occ, req, prio, vic, policy=policy, lo=lo, hi=hi)
    assert np.array_equal(out, want) and np.array_equal(evict, want_ev)
    # the partition is still in force: a placement lands inside it
    res = eng.place_batch(req[req["op"] == E.OP_ALLOC][:1])
    assert res["status"][0] != E.ST_PLACED or lo <= int(res["gpu"][0]) < hi
    eng.close()


def test_state_is_unchanged():
    """Live occupancy, a snapshot, the partition and the stats (all but kernel_launches) are what they were."""
    rng = np.random.default_rng(3)
    G = 4096
    node_off = node_offsets(G // 8, 8)
    rows = E.make_profiles(tables.H100_80GB)
    occ, vic = random_state(rng, G, 1, len(rows))
    eng = engine(node_off, rows, occ)
    eng.place_batch(random_requests(rng, 100, len(rows))[0])
    live = eng.read_occupancy()
    eng.snapshot_occupancy()
    _ = eng.place_batch(random_requests(rng, 50, len(rows))[0])
    moved = eng.read_occupancy()
    before = eng.stats()
    out, _ev = eng.preempt(*random_requests(rng, 200, len(rows)), vic)      # placements only add busy slices: every victim is still valid
    assert (out["status"] == E.ST_PLACED).any()
    after = eng.stats()
    assert np.array_equal(eng.read_occupancy(), moved)
    assert after["kernel_launches"] > before["kernel_launches"]
    for k in before:
        if k != "kernel_launches":
            assert before[k] == after[k], k
    eng.restore_occupancy()
    assert np.array_equal(eng.read_occupancy(), live)
    eng.close()


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_one_request_equals_place_batch(policy, quirks):
    """Rule 5(b): a pod that fits without eviction evicts nothing and gets isl_place_batch's record."""
    rng = np.random.default_rng(17 + policy + quirks)
    G = 4096
    node_off = node_offsets(G // 8, 8)
    names, rows = E.make_profile_tables([tables.A100_40GB, tables.A30_24GB])
    node_table = rng.integers(0, 2, len(node_off) - 1).astype(np.uint8)
    occ, vic = random_state(rng, G, 2, len(names))
    occ |= 0x7F
    occ[rng.integers(0, G, 40)] &= rng.integers(0, 256, 40).astype(np.uint8)
    eng = engine(node_off, rows, occ, policy, quirks, node_table)
    vic = vic[[(occ[v["gpu"]] & PO.span(v["start"], v["size"])) == PO.span(v["start"], v["size"]) for v in vic]]
    for p in range(len(names)):
        req = np.zeros(1, dtype=E.REQUEST_DTYPE)
        req["profile"] = p
        out, evict = eng.preempt(req, np.array([255], np.uint8), vic)
        want = eng.place_batch(req)
        if (evict[0] == E.GPU_NONE).all():
            assert np.array_equal(out, want), (p, out, want)
        else:
            assert want["status"][0] != E.ST_PLACED, p
        if want["status"][0] == E.ST_PLACED:
            eng.free_batch(np.array([(want["gpu"][0], want["start"][0], want["size"][0], 0)], dtype=E.SPAN_DTYPE))
    eng.close()


def code_of(fn):
    try:
        fn()
    except E.EngineError as err:
        return err.code
    return E.OK


def test_error_codes_change_nothing():
    node_off = node_offsets(2, 4)
    rows = E.make_profiles(tables.A100_40GB)
    occ = np.array([0x0F, 0x01, 0, 0, 0, 0, 0, 0], dtype=np.uint8)
    eng = engine(node_off, rows, occ, max_batch=16)
    req = np.zeros(1, dtype=E.REQUEST_DTYPE)
    one = np.ones(1, np.uint8)
    good = np.array([(0, 0, 4, 1, 0)], dtype=E.VICTIM_DTYPE)
    eng.snapshot_occupancy()
    for bad in [(0, 0, 0, 1, 0), (0, 6, 3, 1, 0), (8, 0, 1, 1, 0), (2, 0, 1, 1, 0), (1, 0, 2, 1, 0)]:
        assert code_of(lambda: eng.preempt(req, one, np.array([bad], dtype=E.VICTIM_DTYPE))) == E.EINVAL, bad
    overlap = np.array([(0, 0, 2, 1, 0), (0, 1, 1, 1, 0)], dtype=E.VICTIM_DTYPE)
    assert code_of(lambda: eng.preempt(req, one, overlap)) == E.EINVAL
    free_op = req.copy()
    free_op["op"] = E.OP_FREE
    assert code_of(lambda: eng.preempt(free_op, one, good)) == E.EINVAL
    assert code_of(lambda: eng.preempt(np.zeros(17, dtype=E.REQUEST_DTYPE), np.ones(17, np.uint8), good)) == E.ERANGE
    too_many = np.zeros(8 * 4096 + 1, dtype=E.VICTIM_DTYPE)
    assert code_of(lambda: eng.preempt(req, one, too_many)) == E.ERANGE
    L, h = eng._lib, eng._h
    assert L.isl_preempt(h, 1, None, None, 0, None, None, None) == E.EINVAL
    assert L.isl_preempt(h, 0, None, None, 1, None, None, None) == E.EINVAL
    eng.set_partition(3, 3)
    assert code_of(lambda: eng.preempt(req, one, good)) == E.ERANGE
    eng.set_partition(0, 8)
    # a victim outside the partition is ignored, not refused
    eng.set_partition(1, 8)
    out, _ = eng.preempt(req, one, np.array([(0, 0, 4, 1, 0), (0, 0, 4, 1, 0)], dtype=E.VICTIM_DTYPE))
    assert int(out["gpu"][0]) == 1 and int(out["start"][0]) == 1
    eng.set_partition(0, 8)
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.restore_occupancy()                              # the snapshot survived every refused call
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()
    # ESTATE: no profiles / no inventory, an open stream
    bare = E.Engine(max_gpus=64, max_batch=65536)          # room for one open-stream batch
    assert code_of(lambda: bare.preempt(req, one, good)) == E.ESTATE
    bare.load_profiles(rows)
    assert code_of(lambda: bare.preempt(req, one, good)) == E.ESTATE
    bare.load_inventory(node_off, occ)
    bare.stream_open(1)
    assert code_of(lambda: bare.preempt(req, one, good)) == E.ESTATE
    bare.stream_close()
    bare.close()
    alln = engine(node_off, rows, occ, flags=E.FLAG_ALL_NODES)
    assert code_of(lambda: alln.preempt(req, one, good)) == E.EINVAL
    alln.close()


def test_controller_end_to_end():
    """preempt_pending_pods, then per pod in order: "fits" -> place; "preempt" -> release the victims, place.  Each pod lands exactly
    where it was reported: after the release only V's slices are newly free, the pod fit nowhere before, and rule 5(a) fixes the start."""
    rnd = random.Random(7)
    for trial in range(6):
        items, ranks = random_cluster(rnd, rnd.choice([16, 64]))
        # a homogeneous-quirk controller over the random cluster; priorities as PriorityClass values (int32), some victims deleted
        pod_priority = {u: r * 1000 - 5000 for u, r in ranks.items()}
        for it in items:
            for u, a in it["spec"]["allocations"].items():
                if u in ranks and rnd.random() < 0.05:
                    a["allocationStatus"] = "deleted"
        rec = ctl.InstasliceReconciler(items)
        pods = [{"uid": "pend-%d-%d" % (trial, i), "name": "p%d" % i, "profile": p["profile"], "priority": p["rank"] * 1000 - 4500}
                for i, p in enumerate(random_pods(rnd, items, 12))]
        answers = rec.preempt_pending_pods(pods, pod_priority)
        assert len(answers) == len(pods)
        for pod, (kind, where, gone) in zip(pods, answers):
            if kind == "none":
                continue
            if kind == "preempt":
                for u in gone:
                    assert pod_priority[u] < pod["priority"]
                    assert rec.release(u)
            res = rec.place_pending_pods([pod])[0]
            assert res[0] == "placed", (trial, pod, kind, where, gone, res)
            if kind == "preempt":
                assert (res[1]["gpuUUID"], res[1]["start"], res[1]["size"]) == (where["gpuUUID"], where["start"], where["size"])
                assert res[1]["nodename"] == where["nodename"]


def test_host_mirror_preempt_selftest(tmp_path):
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_preempt_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(root, "tests", "host_mirror_preempt_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
