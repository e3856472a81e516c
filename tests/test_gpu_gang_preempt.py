"""Gang preemption (isl_preempt on an ISL_FLAG_GANG_PREEMPT engine, include/islplace.h P1-P8) on the H100: k_preempt_gangs against the
brute force of tests/gang_preempt_fast.cpp, records and evict rows byte-identical, on random clusters and at the inventory limits; P6
(a)-(c) against the device's own unflagged isl_preempt and isl_place_gangs; the refusals of P1 and P7 in every engine state; the
controller flow and the C++ mirror's self-test."""
import os
import random
import subprocess

import numpy as np
import pytest

from instaslice_b200 import controller as ctl
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import node_offsets

import gang_preempt_fast as GF
import gang_preempt_oracle as GO

pytestmark = pytest.mark.gpu
POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
LOC_FLAGS = {E.GANG_ANY_NODES: 0, E.GANG_ONE_NODE: E.FLAG_GANG_ONE_NODE, E.GANG_DISTINCT_NODES: E.FLAG_GANG_DISTINCT_NODES,
             GO.PER_GANG: E.FLAG_GANG_LOCALITY}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def engine(node_off, rows, occ, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, flags=E.FLAG_GANG_PREEMPT,
           max_batch=4096, lo=None, hi=None):
    eng = E.Engine(max_gpus=max(4096, int(node_off[-1])), max_batch=max_batch, policy=policy, quirks=quirks, flags=flags)
    if rows.ndim == 1:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    if lo is not None:
        eng.set_partition(lo, hi)
    return eng


def device(inputs, flags=E.FLAG_GANG_PREEMPT, max_batch=4096):
    node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc = inputs
    eng = engine(node_off, rows, occ, policy, quirks, node_table, flags | LOC_FLAGS[loc], max_batch, lo, hi)
    try:
        out, evict = eng.preempt(req, prio, vic)
        assert np.array_equal(eng.read_occupancy(), occ)
        return out, evict
    finally:
        eng.close()


def assert_same(inputs, got):
    rc, want, want_ev = GO.run(GF.preempt, inputs)
    assert rc == E.OK
    out, evict = got
    bad = np.flatnonzero((out != want) | (evict != want_ev).any(axis=1))
    assert len(bad) == 0, (bad[:5], out[bad[:5]], want[bad[:5]], evict[bad[:5]], want_ev[bad[:5]])


@pytest.mark.parametrize("case", GO.kat_cases(), ids=lambda c: c["name"])
def test_kat(case):
    inputs = GO.case_inputs(case)
    out, evict = device(inputs)
    recs, ev = GO.expected(case)
    assert [tuple(int(x) for x in r) for r in out] == recs
    assert [[int(k) for k in row if k != E.GPU_NONE] for row in evict] == ev


@pytest.mark.parametrize("loc", [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GO.PER_GANG])
def test_random_clusters(loc):
    """Every policy, both quirk sets, 1-3 tables, partitions that cut nodes, gangs of 1-6 with NOOPs and unknown profiles."""
    rnd = random.Random(100 + loc)
    for it in range(60):
        _names, rows = GO.random_rows(rnd)
        inputs = GO.random_case(rnd, rnd.choice([1, 2, 7, 16, 40]), rnd.randint(1, 24), rows, max_gang=6, locality=loc)
        assert_same(inputs, device(inputs))


def sixteen_profiles_eight_tables(rnd):
    """8 tables of 16 synthetic rows of one start each (the engine takes 128 candidates in all): random sizes 1..7 and starts, so
    that masks of many widths and offsets occur."""
    rows = np.zeros((8, 16), dtype=E.PROFILE_DTYPE)
    for t in range(8):
        for p in range(16):
            size = rnd.randint(1, 7)
            rows[t, p]["size"] = size
            rows[t, p]["n_starts"] = 1
            rows[t, p]["starts"][0] = rnd.randrange(0, 8 - size)
    return rows


@pytest.mark.parametrize("loc", [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GO.PER_GANG])
def test_table_limits(loc):
    rnd = random.Random(7 + loc)
    for it in range(12):
        rows = sixteen_profiles_eight_tables(rnd)
        inputs = GO.random_case(rnd, rnd.choice([7, 33, 120]), rnd.randint(8, 40), rows, max_gang=8, locality=loc)
        assert_same(inputs, device(inputs))


def big_state(rng, G, busy=0.9, listed=0.8):
    """Vectorised random occupancy for large inventories: spans of 1-4 slices, most listed as victims at priorities 0-9 or 255."""
    occ = np.zeros(G, dtype=np.uint8)
    vic = []
    pos = np.zeros(G, dtype=np.int64)
    while True:
        live = np.flatnonzero(pos < 8)
        if len(live) == 0:
            break
        size = np.minimum(rng.integers(1, 5, len(live)), 8 - pos[live])
        b = rng.random(len(live)) < busy
        g, s, z = live[b], pos[live][b], size[b]
        occ[g] |= (((1 << z) - 1) << s).astype(np.uint8)
        keep = rng.random(len(g)) < listed
        pr = np.where(rng.random(len(g)) < 0.05, 255, rng.integers(0, 10, len(g)))
        vic.append(np.rec.fromarrays([g[keep], s[keep], z[keep], pr[keep], np.zeros(keep.sum())], dtype=E.VICTIM_DTYPE))
        pos[live] += size
    vic = np.concatenate(vic).view(E.VICTIM_DTYPE) if vic else np.zeros(0, dtype=E.VICTIM_DTYPE)
    return occ, vic[rng.permutation(len(vic))]


def big_requests(rng, n, n_names, max_gang, prio_hi=12):
    req = np.zeros(n, dtype=E.REQUEST_DTYPE)
    prio = np.zeros(n, dtype=np.uint8)
    i, h = 0, 0
    while i < n:
        k = min(n - i, int(rng.integers(1, max_gang + 1)))
        req["handle"][i:i + k] = h
        req["profile"][i:i + k] = rng.integers(0, n_names, k)
        prio[i:i + k] = rng.integers(1, prio_hi)
        i += k
        h += 1
    req["op"] = E.OP_ALLOC
    return req, prio


@pytest.mark.parametrize("G,nodes_of,n_req,max_gang", [(1, 1, 6, 3), (7, 3, 12, 4), (4096, 8, 64, 8), (65536, 8, 48, 8),
                                                       (65536, 65536, 16, 16), (1 << 20, 8, 12, 4), (1 << 20, 1 << 20, 3, 3)])
@pytest.mark.parametrize("loc", [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES])
def test_inventory_sizes(G, nodes_of, n_req, max_gang, loc):
    """1, 7, 4 096, 65 536 and 2^20 GPUs; nodes of 8 GPUs, and one node of every GPU (a share in global memory at 2^20)."""
    rng = np.random.default_rng(G + nodes_of + loc)
    names, rows = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB])
    node_off = node_offsets(max(1, G // nodes_of), min(nodes_of, G)) if G > 1 else np.array([0, 1], dtype=np.uint32)
    node_off = np.asarray(node_off, dtype=np.uint32)
    node_off[-1] = G
    node_table = (np.arange(len(node_off) - 1) % 2).astype(np.uint8)
    occ, vic = big_state(rng, G)
    req, prio = big_requests(rng, n_req, rows.shape[1], max_gang)
    for policy in ([E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT] if G >= 65536 else POLICIES):
        inputs = (node_off, rows, node_table, occ, req, prio, vic, E.QUIRKS_REF_EXACT, policy, 0, G, loc)
        assert_same(inputs, device(inputs))


def test_cta_layout_edges():
    """Partitions that cut nodes, shares of one node each, nodes larger than a CTA's share (global memory) and empty shares' edges."""
    rng = np.random.default_rng(5)
    names, rows = E.make_profile_tables([tables.A100_40GB])
    for G, sizes in [(600, [1] * 300 + [300]), (9000, [4500, 1, 4499]), (140000, [130000, 10000]), (2048, [1] * 2048)]:
        node_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
        occ, vic = big_state(rng, G)
        for loc in (E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, E.GANG_ANY_NODES):
            req, prio = big_requests(rng, 24, rows.shape[1], 6)
            lo, hi = int(rng.integers(0, G // 3)), int(rng.integers(2 * G // 3, G + 1))
            inputs = (node_off, rows, None, occ, req, prio, vic, E.QUIRKS_FIXED, E.POLICY_FIRST_FIT, lo, hi, loc)
            assert_same(inputs, device(inputs))


@pytest.mark.parametrize("gang", [1, 2, 64, 1024])
def test_large_gangs(gang):
    rng = np.random.default_rng(gang)
    names, rows = E.make_profile_tables([tables.A100_40GB])
    G = 4096
    node_off = np.asarray(node_offsets(G // 512, 512), dtype=np.uint32)
    occ, vic = big_state(rng, G, busy=0.95)
    for loc in (E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES):
        req, prio = big_requests(rng, 2048, rows.shape[1], gang, prio_hi=9)
        inputs = (node_off, rows, None, occ, req, prio, vic, E.QUIRKS_REF_EXACT, E.POLICY_BEST_FIT, 0, G, loc)
        assert_same(inputs, device(inputs))


def test_one_node_key_overflow():
    """A one-node gang of 1 024 members, each evicting 8 victims at priority 200: the node cost's sum (1 638 400) and count (8 192)
    overflow the single-pod key's fields (11 and 4 bits).  Node 1 holds 2-slice victims (count 4 096, sum 819 200) and must win; node 0,
    first in scan order, holds the 8 192 one-slice victims."""
    names, rows = E.make_profile_tables([tables.A100_40GB])
    G = 2048
    node_off = np.array([0, 1024, 2048], dtype=np.uint32)
    occ = np.full(G, 0xFF, dtype=np.uint8)
    vic = [(g, s, 1, 200, 0) for g in range(1024) for s in range(8)] + [(g, s, 2, 200, 0) for g in range(1024, 2048) for s in range(0, 8, 2)]
    vic = np.array(vic, dtype=E.VICTIM_DTYPE)
    req = np.zeros(1024, dtype=E.REQUEST_DTYPE)
    req["profile"] = names.index("7g.40gb")
    req["op"] = E.OP_ALLOC
    prio = np.full(1024, 201, dtype=np.uint8)
    inputs = (node_off, rows, None, occ, req, prio, vic, E.QUIRKS_FIXED, E.POLICY_FIRST_FIT, 0, G, E.GANG_ONE_NODE)
    out, evict = device(inputs)
    assert_same(inputs, (out, evict))
    assert (out["status"] == E.ST_PLACED).all() and (out["gpu"] >= 1024).all()


def test_one_node_count_decides():
    """The first words tie: every victim at priority 0, so both nodes cost (1, 0).  Node 0, first in scan order, would evict 8 192
    one-slice victims, node 1 only 4 096 two-slice victims: only the second word's count, far beyond the single-pod key's 4 bits,
    sends the gang of 1 024 members to node 1."""
    names, rows = E.make_profile_tables([tables.A100_40GB])
    G = 2048
    node_off = np.array([0, 1024, 2048], dtype=np.uint32)
    occ = np.full(G, 0xFF, dtype=np.uint8)
    vic = [(g, s, 1, 0, 0) for g in range(1024) for s in range(8)] + [(g, s, 2, 0, 0) for g in range(1024, 2048) for s in range(0, 8, 2)]
    vic = np.array(vic, dtype=E.VICTIM_DTYPE)
    req = np.zeros(1024, dtype=E.REQUEST_DTYPE)
    req["profile"] = names.index("7g.40gb")
    prio = np.full(1024, 1, dtype=np.uint8)
    inputs = (node_off, rows, None, occ, req, prio, vic, E.QUIRKS_FIXED, E.POLICY_FIRST_FIT, 0, G, E.GANG_ONE_NODE)
    out, evict = device(inputs)
    assert_same(inputs, (out, evict))
    assert (out["status"] == E.ST_PLACED).all() and (out["gpu"] >= 1024).all()
    assert (evict != E.GPU_NONE).sum() == 4096


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT])
def test_one_node_node_index_above_2_20(policy):
    """Empty nodes count as node indices: three GPUs whose winning node has index 2^20 + 1 (gang_preempt_oracle.node_index_case).  A 20-bit node field
    would name node 1, which takes only one of the two members, and commit half a gang."""
    inputs = GO.node_index_case(policy)
    out, evict = device(inputs)
    assert_same(inputs, (out, evict))
    assert out["status"].tolist() == [E.ST_PLACED, E.ST_PLACED] and out["gpu"].tolist() == [2, 2]
    assert (evict == E.GPU_NONE).all()


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("loc", [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES])
def test_gangs_of_one_equal_unflagged(policy, loc):
    """P6 (a): with every handle distinct a flagged call equals the device's unflagged isl_preempt."""
    rnd = random.Random(policy * 10 + loc)
    for it in range(8):
        _n, rows = GO.random_rows(rnd)
        inputs = list(GO.random_case(rnd, rnd.choice([5, 30, 200]), 40, rows, max_gang=1, locality=loc, policy=policy))
        inputs[4] = inputs[4].copy()
        inputs[4]["handle"] = np.arange(len(inputs[4]))
        got = device(tuple(inputs))
        node_off, rows, node_table, occ, req, prio, vic, quirks, policy_, lo, hi, _ = inputs
        eng = engine(node_off, rows, occ, policy_, quirks, node_table, 0, lo=lo, hi=hi)
        want = eng.preempt(req, prio, vic)
        eng.close()
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT])
@pytest.mark.parametrize("loc", [E.GANG_ANY_NODES, E.GANG_ONE_NODE, E.GANG_DISTINCT_NODES, GO.PER_GANG])
def test_no_victims_equal_place_gangs(policy, loc):
    """P6 (b): with no victim below its gang's priority a flagged call returns the records of the device's isl_place_gangs."""
    rnd = random.Random(policy * 7 + loc)
    for it in range(8):
        _n, rows = GO.random_rows(rnd)
        node_off, rows, node_table, occ, req, prio, vic, quirks, _p, lo, hi, _ = GO.random_case(rnd, rnd.choice([6, 40]), 30, rows,
                                                                                             max_gang=5, locality=loc, policy=policy)
        req = req.copy()
        req["profile"][req["profile"] == E.PROFILE_UNKNOWN] = 0
        if it % 2:
            vic = vic[:0]
        else:
            prio = np.minimum(prio, 0).astype(np.uint8)          # every gang at priority 0: no victim is below it
        inputs = (node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc)
        out, evict = device(inputs)
        eng = engine(node_off, rows, occ, policy, quirks, node_table, LOC_FLAGS[loc], lo=lo, hi=hi)
        bounds = GO.gang_bounds(req)
        placed = eng.place_gangs(req, [a for a, _ in bounds] + [len(req)])
        eng.close()
        assert np.array_equal(out, placed)
        assert (evict == E.GPU_NONE).all()


def test_query_changes_nothing():
    """P6 (c): occupancy, snapshot, partition and stats (except kernel_launches) are the same after a call."""
    rnd = random.Random(3)
    _n, rows = GO.random_rows(rnd, 2)
    node_off, rows, node_table, occ, req, prio, vic, quirks, policy, lo, hi, loc = GO.random_case(rnd, 64, 40, rows, locality=GO.PER_GANG)
    eng = engine(node_off, rows, occ, policy, quirks, node_table, E.FLAG_GANG_PREEMPT | E.FLAG_GANG_LOCALITY, lo=8, hi=56)
    eng.snapshot_occupancy()
    before = eng.stats()
    eng.preempt(req, prio, vic)
    after = eng.stats()
    assert np.array_equal(eng.read_occupancy(), occ)
    assert {k: v for k, v in before.items() if k != "kernel_launches"} == {k: v for k, v in after.items() if k != "kernel_launches"}
    out, _ = eng.preempt(req, prio, vic)
    rc, want, _ = GO.run(GF.preempt, (node_off, rows, node_table, occ, req, prio, vic, quirks, policy, 8, 56, loc))
    assert np.array_equal(out, want)                              # the partition stayed in place
    eng.write_occupancy(0, np.zeros(len(occ), dtype=np.uint8))
    eng.restore_occupancy()
    assert np.array_equal(eng.read_occupancy(), occ)              # the snapshot survived
    eng.close()


def code_of(fn):
    try:
        fn()
    except E.EngineError as ex:
        return ex.code
    return E.OK


def _state(eng):
    """What a refused call must leave as it was: the occupancy and every stat except kernel_launches."""
    st = {k: v for k, v in eng.stats().items() if k != "kernel_launches"}
    return eng.read_occupancy(), st


def test_refusals():
    """P7 at isl_create; P1's EINVAL and rule 2's victim checks, each leaving the occupancy and stats as they were; isl_preempt's code in
    every engine state of a flagged engine, the three open-stream sub-states included (opened, a batch in, every batch in and waited);
    after them the occupancy, the snapshot and the partition are unchanged."""
    for extra in (E.FLAG_ALL_NODES, E.FLAG_GANG_FEW_NODES, E.FLAG_GANG_MIN_MEMBERS):
        assert code_of(lambda: E.Engine(64, 64, flags=E.FLAG_GANG_PREEMPT | extra)) == E.EINVAL
    for policy in (E.POLICY_MOST_ALLOCATED, E.POLICY_LEAST_ALLOCATED):
        E.Engine(64, 64, policy=policy, flags=E.FLAG_GANG_PREEMPT).close()
    names, rows = E.make_profile_tables([tables.A100_40GB])
    req = np.zeros(2, dtype=E.REQUEST_DTYPE)
    req["profile"] = names.index("1g.5gb")
    two = np.array([3, 3], dtype=np.uint8)
    vic = np.array([(0, 0, 1, 1, 0)], dtype=E.VICTIM_DTYPE)
    occ = np.array([1, 0, 0, 0], dtype=np.uint8)
    node_off = np.array([0, 2, 4], dtype=np.uint32)
    eng = E.Engine(64, 2 * 65536, flags=E.FLAG_GANG_PREEMPT | E.FLAG_GANG_LOCALITY)  # room for two open-stream batches
    assert code_of(lambda: eng.preempt(req, two, vic)) == E.ESTATE            # created
    eng.load_profile_tables(rows)
    assert code_of(lambda: eng.preempt(req, two, vic)) == E.ESTATE            # profiles only
    eng2 = E.Engine(64, 64, flags=E.FLAG_GANG_PREEMPT)
    eng2.load_inventory(node_off, occ)
    assert code_of(lambda: eng2.preempt(req, two, vic)) == E.ESTATE           # inventory only
    assert np.array_equal(eng2.read_occupancy(), occ)
    eng2.close()
    eng.load_inventory(node_off, occ)
    eng.set_partition(0, 3)
    eng.snapshot_occupancy()
    before = _state(eng)

    def refused(code, r, pr, v=vic):
        assert code_of(lambda: eng.preempt(r, pr, v)) == code
        after = _state(eng)
        assert np.array_equal(after[0], before[0]) and after[1] == before[1]

    refused(E.EINVAL, req, np.array([3, 4], dtype=np.uint8))                 # two priorities in one gang
    for a, b in ((0, 1), (1, 3), (2, 2), (4, 4)):
        r2 = req.copy()
        r2["start"] = (a, b)
        refused(E.EINVAL, r2, two)                                            # two localities, few nodes or a byte above 3
    r2 = req.copy()
    r2["handle"] = (0, 1)
    r2["start"] = (2, 0)
    refused(E.EINVAL, r2, two)
    refused(E.EINVAL, req, two, np.array([(1, 0, 1, 1, 0)], dtype=E.VICTIM_DTYPE))         # a victim on a free slice (rule 2)
    refused(E.EINVAL, req, two, np.array([(0, 0, 1, 1, 0), (0, 0, 1, 2, 0)], dtype=E.VICTIM_DTYPE))   # overlapping victims
    refused(E.EINVAL, req, two, np.array([(9, 0, 1, 1, 0)], dtype=E.VICTIM_DTYPE))         # gpu >= G
    r2["op"][0] = E.OP_NOOP                                                   # a NOOP's bytes are not looked at
    out, _ = eng.preempt(r2, np.array([9, 3], dtype=np.uint8), vic)
    assert tuple(out["status"]) == (E.ST_NOOP, E.ST_PLACED)
    r2["op"][0] = E.OP_FREE
    refused(E.EINVAL, r2, two)                                                # rule 3
    with pytest.raises(ValueError):
        E.Engine(64, 64).preempt(req, two, vic, gang_off=[0, 2])
    eng.set_partition(2, 2)
    assert code_of(lambda: eng.preempt(req, two, vic)) == E.ERANGE            # empty partition
    eng.set_partition(0, 3)
    assert np.array_equal(eng.read_occupancy(), occ)
    noop = E.PinnedArray(2 * 16, E.REQUEST_DTYPE)                             # NOOP batches: the stream itself changes nothing
    res = E.PinnedArray(2 * 16, E.RESULT_DTYPE)
    noop.array[:] = np.zeros(32, dtype=E.REQUEST_DTYPE)
    noop.array["op"] = E.OP_NOOP
    for sub in ("opened", "one batch in", "every batch in"):
        eng.stream_open(2)
        try:
            for b in range({"opened": 0, "one batch in": 1, "every batch in": 2}[sub]):
                eng.stream_wait(eng.stream_submit_ptr(16, noop.ptr + 8 * 16 * b, res.ptr + 8 * 16 * b))
            assert code_of(lambda: eng.preempt(req, two, vic)) == E.ESTATE, sub
            assert code_of(lambda: eng.preempt(req, np.array([3, 4], dtype=np.uint8), vic)) == E.EINVAL, sub   # argument checks first
        finally:
            eng.stream_close()
        assert np.array_equal(eng.read_occupancy(), occ), sub
    noop.free()
    res.free()
    out, evict = eng.preempt(req, two, vic)                                   # the partition [0, 3) is still in place
    assert tuple(out["status"]) == (E.ST_PLACED, E.ST_PLACED)
    assert set(out["gpu"].tolist()) <= {0, 1, 2}
    eng.write_occupancy(0, np.full(4, 0xFF, dtype=np.uint8))
    eng.restore_occupancy()                                                   # the snapshot survived every refused call
    assert np.array_equal(eng.read_occupancy(), occ)
    eng.close()


def test_controller_flow():
    """preempt_pending_gangs -> delete the union of the victims -> place_pending_gangs places the gang where it was shown: the one-node
    gang of two 3g.20gb takes the node with two cheap victims over the node with one more important one."""
    import preempt_oracle as PO
    case = {"tables": ["a100-40gb"], "node_off": [0, 1, 2], "node_table": [0, 0], "occ": [255, 255],
            "victims": [[0, 0, 8, 3], [1, 0, 4, 1], [1, 4, 4, 2]]}
    items = PO.case_items(case)
    rc = ctl.InstasliceReconciler(items, quirks=E.QUIRKS_FIXED, gang_preempt=True, gang_one_node=True)
    gang = [{"uid": "w%d" % i, "name": "w%d" % i, "profile": "3g.20gb", "priority": 50} for i in range(2)]
    prios = {"v0": 30, "v1": 10, "v2": 20}
    kind, where, gone = rc.preempt_pending_gangs([gang], prios)[0]
    assert kind == "preempt" and gone == ["v1", "v2"]
    assert [(w["gpuUUID"], w["start"], w["size"]) for w in where] == [("GPU-000001", 0, 4), ("GPU-000001", 4, 4)]
    for uid in gone:
        assert rc.release(uid)
    placed = rc.place_pending_gangs([gang])
    assert placed[0][0] == "placed"
    assert [(a["gpuUUID"], a["start"]) for a in placed[0][1]] == [("GPU-000001", 0), ("GPU-000001", 4)]
    assert rc.preempt_pending_gangs([[dict(gang[0], uid="x")]], prios)[0][0] in ("preempt", "none")
    with pytest.raises(ValueError):
        rc.preempt_pending_gangs([[dict(gang[0], priority=1), gang[1]]], prios)
    plain = ctl.InstasliceReconciler(PO.case_items(case), quirks=E.QUIRKS_FIXED)
    with pytest.raises(ValueError):
        plain.preempt_pending_gangs([gang], prios)


def test_host_mirror_selftest(tmp_path):
    pkg = os.path.join(ROOT, "instaslice_b200")
    exe = str(tmp_path / "host_mirror_gang_preempt_selftest")
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "host_mirror_gang_preempt_selftest.cpp"),
                    "-L" + pkg, "-l:libislhost.so", "-l:libislplace.so", "-Wl,-rpath," + pkg], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "PASS" in out.stdout, out.stdout + out.stderr
