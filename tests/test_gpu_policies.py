"""SURVEY 8f-4 behind the allocation-policy hook: GPU-order right-to-left (the reference's stub, :464-469), the pairs-lost
fragmentation scorer, the what-if query, per-profile capacity, and the literal no-`break` node loop (Q5) — each against the CPU
oracle through the C ABI.  Needs an H100."""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables, workloads as W

from range_oracle import capacity_by_hand

pytestmark = pytest.mark.gpu


def _churn(rng, ref, sizes, n_profiles):
    batches, live = [], []
    for n in sizes:
        req = W.alloc_requests((rng.next(n) % np.uint64(n_profiles)).astype(np.uint8))
        for _ in range(min(len(live), n // 3)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        res = ref.place(req)
        for r in res[(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)]:
            live.append((int(r["gpu"]), int(r["start"]), int(r["size"])))
        batches.append((req, res))
    return batches


@pytest.mark.parametrize("G,flags", [(8, 0), (520, 0), (4096, 0), (4096, E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL), (65536, 0), (20000, E.FLAG_FORCE_PIPELINE)])
def test_right_to_left_gpu_order_vs_oracle(G, flags):
    """ISL_POLICY_RIGHT_TO_LEFT = first-fit over the GPUs in descending canonical order; every device path (k_few, k_small, single
    chain, scan mode, segment pipeline, stream) reports canonical GPU indices and takes canonical FREEs."""
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(31 + G)
    node_off = np.concatenate([[0], np.cumsum(np.full((G + 7) // 8, 8))]).astype(np.uint32)
    node_off[-1] = G
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows, 3, policy=E.POLICY_RIGHT_TO_LEFT)
    ref.load(occ)
    sizes = [3, 1, 700, 5000, 70000, 8, 1500] if G >= 4096 else [3, 1, 40, 700, 8]
    batches = _churn(rng, ref, sizes, len(rows))
    eng = E.Engine(max_gpus=max(4096, G), max_batch=1 << 18, policy=E.POLICY_RIGHT_TO_LEFT, flags=flags)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    assert np.array_equal(eng.read_occupancy(), occ)
    for i, (req, want) in enumerate(batches):
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (i, bad[:5], got[bad[:5]], want[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    # the same batches as ONE stream call on a fresh inventory
    eng.load_inventory(node_off, occ)
    got = eng.place_stream([b[0] for b in batches])
    assert all(np.array_equal(a, b[1]) for a, b in zip(got, batches))
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    # write_occupancy / place_batch_range / free_batch speak canonical indices too
    eng.write_occupancy(3, np.array([0x7F, 0x00], dtype=np.uint8))
    o = eng.read_occupancy()
    assert o[3] == 0x7F and o[4] == 0x00
    if G >= 16:
        res = eng.place_batch_range(0, 8, W.alloc_requests(np.zeros(1, dtype=np.uint8)))
        if res["status"][0] == E.ST_PLACED:
            assert int(res["gpu"][0]) < 8
            spans = np.zeros(1, dtype=E.SPAN_DTYPE)
            spans[0] = (res["gpu"][0], res["start"][0], res["size"][0], 0)
            eng.free_batch(spans)
            assert np.array_equal(eng.read_occupancy(), o)
    eng.close()


def test_right_to_left_heterogeneous_tables():
    names, rows2d = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
    rng = W.SplitMix64(77)
    n_nodes = 96
    node_off = W.node_offsets(n_nodes, 8)
    G = n_nodes * 8
    node_table = (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows2d, 3, policy=E.POLICY_RIGHT_TO_LEFT, node_table=node_table)
    ref.load(occ)
    batches = _churn(rng, ref, [5, 300, 2500], len(names))
    eng = E.Engine(max_gpus=4096, max_batch=1 << 16, policy=E.POLICY_RIGHT_TO_LEFT)
    eng.load_profile_tables(rows2d)
    eng.load_inventory(node_off, occ)
    eng.set_node_tables(node_table)
    for i, (req, want) in enumerate(batches):
        assert np.array_equal(eng.place_batch(req), want), i
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    eng.close()


@pytest.mark.parametrize("G,table", [(64, tables.A100_40GB), (2048, tables.H100_80GB), (6000, tables.H100_80GB)])
def test_min_frag_policy_vs_oracle(G, table):
    """ISL_POLICY_MIN_FRAG: the feasible GPU where the placement makes the fewest (profile, start) pairs infeasible, ties to the lowest
    index.  The oracle counts the pairs one by one from the rows; the engine uses a per-byte score table."""
    rows = E.make_profiles(table)
    rng = W.SplitMix64(5 + G)
    node_off = W.node_offsets(G // 8, 8)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows, 3, policy=E.POLICY_MIN_FRAG)
    ref.load(occ)
    batches = _churn(rng, ref, [7, 200, 1200] if G > 64 else [7, 60], len(rows))
    eng = E.Engine(max_gpus=max(4096, G), max_batch=1 << 16, policy=E.POLICY_MIN_FRAG)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    for i, (req, want) in enumerate(batches):
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (i, bad[:5], got[bad[:5]], want[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    eng.close()


def test_capacity_and_what_if_query():
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(99)
    G = 4096
    node_off = W.node_offsets(G // 8, 8)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    eng = E.Engine(max_gpus=G, max_batch=1 << 16)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    assert np.array_equal(eng.capacity(), capacity_by_hand(rows, 3, occ))
    # plan: release 200 busy spans, then ask for 3000 mixed pods
    ref = oracle.Fast(node_off, rows)
    ref.load(occ)
    busy = np.flatnonzero(occ & 1)[:200]
    plan = W.alloc_requests(W.mix_profiles(rng, 3200))
    for i, g in enumerate(busy):
        plan[i] = (g, 0, E.OP_FREE, 0, 1)
    want = ref.place(plan)
    got, before, after = eng.what_if(plan)
    assert np.array_equal(got, want)
    assert np.array_equal(before, capacity_by_hand(rows, 3, occ))
    assert np.array_equal(after, capacity_by_hand(rows, 3, ref.occupancy()))
    assert np.array_equal(eng.read_occupancy(), occ)            # the live state is back
    # and the engine goes on from the LIVE state
    req = W.alloc_requests(W.mix_profiles(rng, 500))
    ref2 = oracle.Fast(node_off, rows)
    ref2.load(occ)
    assert np.array_equal(eng.place_batch(req), ref2.place(req))
    # an empty plan is a pure measurement
    _, b2, a2 = eng.what_if(np.zeros(0, dtype=E.REQUEST_DTYPE))
    assert np.array_equal(b2, a2)
    eng.close()


@pytest.mark.parametrize("n_nodes,gpn,n", [(4, 2, 30), (16, 8, 400), (6, 1, 5)])
def test_all_nodes_flag_reproduces_the_missing_break(n_nodes, gpn, n):
    """ISL_FLAG_ALL_NODES vs the structure-for-structure oracle with all_nodes=True (Reconcile :190-227 has no `break`): a pod is
    allocated on every node that has capacity; the record names the first node; the occupancy shows all of them."""
    rows = E.make_profiles(tables.A100_40GB)
    rng = W.SplitMix64(n_nodes * 100 + n)
    node_off = W.node_offsets(n_nodes, gpn)
    G = n_nodes * gpn
    occ = ((rng.next(G) & rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    f = oracle.Faithful(node_off, rows)
    f.load_occupancy_as_dangling(occ)
    eng = E.Engine(max_gpus=4096, max_batch=1 << 12, flags=E.FLAG_ALL_NODES)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    for rep in range(2):
        req = W.alloc_requests((rng.next(n) % np.uint64(len(rows))).astype(np.uint8))
        want = f.place(req, all_nodes=True)
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (rep, bad[:5], got[bad[:5]], want[bad[:5]])
        assert np.array_equal(eng.read_occupancy(), f.occupancy()), rep
    # without the flag the same engine input consumes capacity on ONE node per pod
    eng2 = E.Engine(max_gpus=4096, max_batch=1 << 12)
    eng2.load_profiles(rows)
    eng2.load_inventory(node_off, occ)
    f2 = oracle.Faithful(node_off, rows)
    f2.load_occupancy_as_dangling(occ)
    req = W.alloc_requests((rng.next(n) % np.uint64(len(rows))).astype(np.uint8))
    assert np.array_equal(eng2.place_batch(req), f2.place(req, all_nodes=False))
    eng.close(); eng2.close()


@pytest.mark.parametrize("policy", [E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG])
def test_best_fit_family_with_per_node_tables_and_large_inventories(policy):
    """The best-fit family groups the GPUs by (table of the node, occupancy byte): heterogeneous clusters and inventories far beyond
    65 536 GPUs (class bitmaps in global memory) against the oracle's O(G)-per-request search."""
    names, rows2d = E.make_profile_tables([tables.A100_40GB, tables.H100_80GB, tables.A30_24GB])
    rng = W.SplitMix64(1234 + policy)
    n_nodes = 700
    node_off = W.node_offsets(n_nodes, 8)
    G = n_nodes * 8
    node_table = (rng.next(n_nodes) % np.uint64(3)).astype(np.uint8)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows2d, 3, policy=policy, node_table=node_table)
    ref.load(occ)
    batches = _churn(rng, ref, [9, 400, 1500], len(names))
    eng = E.Engine(max_gpus=8192, max_batch=1 << 16, policy=policy)
    eng.load_profile_tables(rows2d)
    eng.load_inventory(node_off, occ)
    eng.set_node_tables(node_table)
    for i, (req, want) in enumerate(batches):
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (i, bad[:5], got[bad[:5]], want[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    eng.close()
    # one table, 200 000 GPUs
    rows = E.make_profiles(tables.H100_80GB)
    G = 200_000
    node_off = W.node_offsets(G // 8, 8)
    occ = ((rng.next(G) | rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows, 3, policy=policy)
    ref.load(occ)
    batches = _churn(rng, ref, [5, 250, 250], len(rows))
    eng = E.Engine(max_gpus=G, max_batch=1 << 16, policy=policy)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    for i, (req, want) in enumerate(batches):
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (i, bad[:5], got[bad[:5]], want[bad[:5]])
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    eng.close()
