"""Every mechanism that joins the ranks of a partitioned inventory, at its limits, on one H100: the token ring, owner-gathered results
with a causal window, the speculative ring and the host-carried token, over worlds of 2 to 8 engines in one process (wired the way
the multi-GPU run wires them through CUDA IPC).  The inputs and every expected byte come from ``test_oracle_partition_limits.py``:
each rank's own result array, the merged MIN, rank 0's gathered array, the WHOLE occupancy of every engine (bytes outside a rank's
range stay as loaded), and the path that ran (``ring_plan``: speculative rounds or not, and every rank's pipeline resident at once
within half of the device's SMs).
"""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W
from range_oracle import RangeFast
from test_oracle_partition_limits import (SPEC_RING_IDS, _Ref, dflt_of, inventory, rank_occupancy, rank_records, ring_plan,
                                          ring_requests, stage_size, total_ctas, trap_tables)
from test_oracle_table_limits import candidates, t8tab, t16x8

pytestmark = pytest.mark.gpu

MULTI = [3000, 0, 70_000, 500]          # an empty batch between non-empty ones, a batch of two chunks


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def fixture(name):
    """(rows, quirks): T8tab (8 node tables) under FIXED quirks, T16x8 or the H100 table under the reference's."""
    return {"t8tab": (t8tab(), E.QUIRKS_FIXED), "t16x8": (t16x8(), E.QUIRKS_REF_EXACT),
            "h100": (E.make_profiles(tables.H100_80GB), E.QUIRKS_REF_EXACT)}[name]


def device_view(ptr, n):
    import torch

    class _View:            # torch view of an engine-owned result array (no copy)
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_View(), device="cuda")


class Ring:
    """world engines over one inventory, engine r owning [bounds[r], bounds[r + 1])."""

    def __init__(self, rows, quirks, node_off, occ, bounds, node_table=None, owner=False, window=0, spec=None, max_batch=1 << 17):
        self.rows, self.quirks, self.node_off, self.occ, self.b, self.node_table = rows, quirks, node_off, occ, bounds, node_table
        self.owner, self.world = owner, len(bounds) - 1
        G = int(node_off[-1])
        self.engines = []
        for _ in range(self.world):
            eng = E.Engine(max_gpus=max(4096, G), max_batch=max_batch, quirks=quirks)
            if rows.ndim == 2:
                eng.load_profile_tables(rows)
            else:
                eng.load_profiles(rows)
            eng.ipc_inbox_handle()
            if spec is not None:
                eng.ipc_spec_handle()
            self.engines.append(eng)
        self.reload()
        for r, eng in enumerate(self.engines):
            eng.connect_local(self.engines[r + 1] if r + 1 < self.world else None, has_prev=r > 0)
            if owner:
                eng.connect_owner_local(self.engines[0] if r > 0 else None)
            if owner or spec is not None:
                eng.set_ring_world(self.world)
            eng.set_causal_window(window)
            if spec is not None:
                eng.connect_spec_local(self.world, r, self.engines, bounds)
                eng.set_speculation(spec)

    def reload(self):
        for eng, lo, hi in zip(self.engines, self.b, self.b[1:]):
            eng.load_inventory(self.node_off, self.occ)
            if self.node_table is not None:
                eng.set_node_tables(self.node_table)
            eng.set_partition(lo, hi)

    def stats(self):
        return [eng.stats() for eng in self.engines]

    def close(self):
        for eng in self.engines:
            eng.close()


def expected(ring, batches):
    ref = oracle.Fast(ring.node_off, ring.rows, ring.quirks, node_table=ring.node_table)
    ref.load(ring.occ)
    return [ref.place(req) for req in batches], ref.occupancy()


def check_ranks(ring, batches, outs, want, final, what, owner_out=None):
    """Each rank's own array, the merged MIN, rank 0's gathered array and every engine's whole occupancy."""
    dflt = dflt_of(ring.rows, ring.node_off, ring.node_table)
    all_want = np.concatenate(want)
    for r, (out, lo, hi) in enumerate(zip(outs, ring.b, ring.b[1:])):
        if owner_out is not None and r == 0:
            mine = all_want
        else:
            mine = np.concatenate([rank_records(req, w, lo, hi, dflt) for req, w in zip(batches, want)])
        bad = np.flatnonzero(out != mine)
        assert len(bad) == 0, (what, r, (lo, hi), bad[:5], out[bad[:5]], mine[bad[:5]])
    if owner_out is None:
        merged = np.minimum.reduce([o.view(np.int64) for o in outs]).view(E.RESULT_DTYPE)
        assert np.array_equal(merged, all_want), what
    for r, (eng, lo, hi) in enumerate(zip(ring.engines, ring.b, ring.b[1:])):
        assert np.array_equal(eng.read_occupancy(), rank_occupancy(ring.occ, final, lo, hi)), (what, r, (lo, hi))


def run_ring(ring, batches, stream_id):
    """One isl_place_stream_partitioned on every rank, ranks launched in order.  Returns every rank's own records."""
    import torch
    sizes = np.array([len(b) for b in batches], dtype=np.uint32)
    total = int(sizes.sum())
    d_in = torch.from_numpy(np.concatenate(batches).view(np.int64).copy()).cuda()
    if ring.owner:
        ptrs = [eng.device_results() for eng in ring.engines]
    else:
        bufs = [torch.full((total,), -1, dtype=torch.int64, device="cuda") for _ in ring.engines]
        ptrs = [b.data_ptr() for b in bufs]
    torch.cuda.synchronize()
    for eng, p in zip(ring.engines, ptrs):
        eng.place_stream_partitioned(sizes, d_in.data_ptr(), p, stream_id)
    for eng in ring.engines:
        eng.synchronize()
    return [device_view(p, total).cpu().numpy().view(E.RESULT_DTYPE).copy() for p in ptrs]


def ring_case(ring, rng, sizes, stream_id, plan, what):
    G = int(ring.node_off[-1])
    batches = ring_requests(rng, _Ref(ring.node_off, ring.rows, ring.quirks, ring.node_table, ring.occ), sizes, ring.rows.shape[-1], G)
    want, final = expected(ring, batches)
    ring.reload()
    before = ring.stats()
    outs = run_ring(ring, batches, stream_id)
    after = ring.stats()
    check_ranks(ring, batches, outs, want, final, what, owner_out=ring.owner or None)
    launches = [a["kernel_launches"] - b["kernel_launches"] for a, b in zip(after, before)]
    spec = [a["spec_chunks"] - b["spec_chunks"] for a, b in zip(after, before)]
    assert launches == [3] * ring.world, (what, launches)            # k_prepare, k_partition, k_pipeline on every rank
    if plan[0] == "spec":
        assert spec[-1] > 0, (what, spec)
    else:
        assert spec == [0] * ring.world, (what, spec)


def planned(ring, sizes, **kw):
    n_cand = len(candidates(ring.rows, ring.quirks))
    p = ring_plan(int(ring.node_off[-1]), ring.b, sizes, n_cand, sms=sm_count(), **kw)
    assert p[0] != "erange" and total_ctas(p) <= sm_count() // 2, p
    return p


# ---- 1. token ring ---------------------------------------------------------------------------------------------------------------------
TOKEN_CASES = [(2, "single", "t16x8"), (3, "word", "t8tab"), (4, "node", "h100"), (5, "unequal", "t8tab"), (6, "proportional", "h100"),
               (7, "word", "t8tab"), (8, "single", "t16x8"), (8, "word", "t8tab")]


@pytest.mark.parametrize("world,kind,table", TOKEN_CASES)
def test_token_ring(world, kind, table):
    rows, quirks = fixture(table)
    node_off, occ, b = inventory(300 + world, world, kind)
    node_table = trap_tables(W.SplitMix64(world), node_off, b) if rows.ndim == 2 else None
    ring = Ring(rows, quirks, node_off, occ, b, node_table)
    rng = W.SplitMix64(40 + world)
    plan = planned(ring, MULTI)
    assert plan[0] == "plain"
    for stream_id in (1, 2):
        ring_case(ring, rng, MULTI, stream_id, plan, (world, kind, table, stream_id))
    ring.close()


# ---- 2. owner-gathered results with the ring's causal window ----------------------------------------------------------------------------
@pytest.mark.parametrize("world,window", [(2, 0), (3, 1), (5, 2), (8, 3)])
def test_owner_gathered_ring(world, window):
    rows, quirks = fixture("t8tab")
    node_off, occ, b = inventory(500 + world, world, "word")
    ring = Ring(rows, quirks, node_off, occ, b, trap_tables(W.SplitMix64(world), node_off, b), owner=True, window=window)
    rng = W.SplitMix64(60 + world)
    plan = planned(ring, MULTI, ring_world=world, window=window)
    for stream_id in (11, 12):
        ring_case(ring, rng, MULTI, stream_id, plan, (world, window, stream_id))
    ring.close()


# ---- 3. speculative ring -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_speculative_ring_on_and_off_the_stage_size(world):
    """Unequal ranks on multiples of the stage size speculate; the same inputs with one bound off it take the plain ring; the records
    are the oracle's either way."""
    rows, quirks = fixture("t8tab" if world % 2 else "t16x8")
    node_off, occ, b = inventory(700 + world, world, "sz")
    off = list(b)
    off[max(1, world // 2)] += 1 + stage_size(int(node_off[-1])) // 2
    node_table = trap_tables(W.SplitMix64(world), node_off, b) if rows.ndim == 2 else None
    sizes = [5000, 0, 3000]
    for bounds, want_path, sid in ((b, "spec", 21), (off, "plain", 22)):
        ring = Ring(rows, quirks, node_off, occ, bounds, node_table, spec=E.SPEC_ON)
        plan = planned(ring, sizes, spec_world=world, ring_world=world, mode="on")
        assert plan[0] == want_path, (bounds, plan)
        ring_case(ring, W.SplitMix64(80 + world), sizes, sid, plan, (world, want_path))
        ring.close()


def test_speculative_ring_64_chunks_and_65():
    rows, quirks = fixture("t8tab")
    node_off, occ, b = inventory(907, 3, "sz")
    ring = Ring(rows, quirks, node_off, occ, b, trap_tables(W.SplitMix64(3), node_off, b), spec=E.SPEC_ON)
    for n_chunks, want_path, sid in ((64, "spec", 31), (65, "plain", 32)):
        sizes = [150] * n_chunks
        plan = planned(ring, sizes, spec_world=3, ring_world=3, mode="on")
        assert plan[0] == want_path
        ring_case(ring, W.SplitMix64(n_chunks), sizes, sid, plan, n_chunks)
    ring.close()


# ---- 4. host-carried token ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [3, 5, 8])
def test_host_carried_token(world):
    import torch
    rows, quirks = fixture("t8tab")
    node_off, occ, b = inventory(1100 + world, world, "word")
    ring = Ring(rows, quirks, node_off, occ, b, trap_tables(W.SplitMix64(world), node_off, b))
    G = int(node_off[-1])
    batches = ring_requests(W.SplitMix64(world), _Ref(node_off, rows, quirks, ring.node_table, occ), [70_000, 2000], 16, G)
    want, final = expected(ring, batches)
    outs = [[] for _ in range(world)]
    for req in batches:
        n = len(req)
        n_chunks = -(-n // 65536)
        d_in = torch.from_numpy(req.view(np.int64).copy()).cuda()
        heads = [torch.full((n_chunks * 16,), -1, dtype=torch.int32, device="cuda") for _ in range(world)]
        for r, eng in enumerate(ring.engines):
            d_out = torch.full((n,), -1, dtype=torch.int64, device="cuda")
            before = eng.stats()["kernel_launches"]
            eng.place_batch_partitioned(n, d_in.data_ptr(), d_out.data_ptr(), heads[r - 1].data_ptr() if r else None, heads[r].data_ptr())
            eng.synchronize()
            assert eng.stats()["kernel_launches"] - before == 1 + 5 * n_chunks
            outs[r].append(d_out.cpu().numpy().view(E.RESULT_DTYPE))
    check_ranks(ring, batches, [np.concatenate(o) for o in outs], want, final, ("host token", world))
    ring.close()


# ---- 5. stream ids -------------------------------------------------------------------------------------------------------------------------
def test_stream_id_boundaries_on_the_speculative_ring():
    """Ids below 2^24 speculate; 2^24 (record tag 0), s + 2^24 after s, and 2^32 - 1 take the token ring; 32 768 shares 1's inbox
    tag.  Every call has its own batches, and each is the oracle's."""
    rows, quirks = fixture("t16x8")
    node_off, occ, b = inventory(1300, 4, "sz")
    ring = Ring(rows, quirks, node_off, occ, b, spec=E.SPEC_ON)
    rng = W.SplitMix64(1300)
    sizes = [4000, 0, 2500]
    for sid in (1, 32767, 32768, SPEC_RING_IDS - 1, SPEC_RING_IDS, 5, 5 + SPEC_RING_IDS, 2 ** 32 - 1):
        plan = planned(ring, sizes, spec_world=4, ring_world=4, mode="on", stream_id=sid)
        assert (plan[0] == "spec") == (sid < SPEC_RING_IDS)
        ring_case(ring, rng, sizes, sid, plan, sid)
    # an engine whose record memory is shared keeps the plain pipeline for its own calls: they would tag with its epoch
    eng, lo, hi = ring.engines[-1], b[-2], b[-1]
    occ_now = eng.read_occupancy()
    req = ring_requests(rng, _Ref(node_off, rows, quirks, None, occ), [6000], 16, int(node_off[-1]))[0]
    ref = RangeFast(node_off, rows, occ_now, lo, hi, quirks)
    before = eng.stats()["spec_chunks"]
    assert np.array_equal(eng.place_batch(req), ref.place(req))
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    assert eng.stats()["spec_chunks"] == before
    ring.close()


# ---- 6. refusals ---------------------------------------------------------------------------------------------------------------------------
def _code(fn):
    try:
        fn()
        return E.OK
    except E.EngineError as e:
        return e.code


@pytest.mark.parametrize("what", ["chunks", "masks", "id0", "bestfit", "rtl", "nodescore"])
def test_refusals_change_nothing(what):
    """On a first rank without a window or speculation (a wrongly accepted call could not wait on another rank)."""
    import torch
    rows, quirks = fixture("h100")
    node_off, occ, b = inventory(1500, 2, "word")
    G = int(node_off[-1])
    policy = {"bestfit": E.POLICY_BEST_FIT, "rtl": E.POLICY_RIGHT_TO_LEFT, "nodescore": E.POLICY_MOST_ALLOCATED}.get(what, E.POLICY_FIRST_FIT)
    max_gpus = (1 << 24) if what == "masks" else max(4096, G)
    sizes = {"chunks": [1] * 4095 + [65537], "masks": [10] * 17}.get(what, [3000, 500])
    total = sum(sizes)
    eng = E.Engine(max_gpus=max_gpus, max_batch=max(total, 1 << 12), quirks=quirks, policy=policy)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    eng.set_partition(b[0], b[1])
    eng.ipc_inbox_handle()
    n_cand = len(candidates(rows, quirks))
    if what in ("chunks", "masks"):
        assert ring_plan(G, b, sizes, n_cand, max_gpus=max_gpus) == ("erange", None)
    req = W.alloc_requests((np.arange(total) % 7).astype(np.uint8))
    d_in = torch.from_numpy(req.view(np.int64).copy()).cuda()
    d_out = torch.full((total,), 0x5555, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    sid = 0 if what == "id0" else 7
    want = {"chunks": E.ERANGE, "masks": E.ERANGE}.get(what, E.EINVAL)
    before = eng.stats()["kernel_launches"]
    assert _code(lambda: eng.place_stream_partitioned(np.array(sizes, dtype=np.uint32), d_in.data_ptr(), d_out.data_ptr(), sid)) == want
    eng.synchronize()
    assert eng.stats()["kernel_launches"] == before
    assert (d_out.cpu().numpy() == 0x5555).all()
    assert np.array_equal(eng.read_occupancy()[:G], occ)
    eng.close()
