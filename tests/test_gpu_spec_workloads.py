"""The structured workloads of spec_workloads.py through the device: the speculative rounds (SPEC_ON, traced), the plain pipeline
(SPEC_OFF) and the default route, batch by batch; multi-batch workloads also as device streams with causal windows 1 and 3; the four
hardest as an open stream; a subset on 2 and 3 ranks of one GPU.  Every result record and the final occupancy are compared byte for byte
with ``oracle.Fast``.

Every traced speculative call is also held to what the rounds promise, per chunk, from the per-cell trace (word 6 decisions, 7
simulations of the cell, 11 its certification round): the cell of global stage 0 is certified in round 1, certification rounds never
decrease along the stages (over all ranks in rank order), no round exceeds stages + 2, a cell simulates at most once per round and at
least once when it placed anything, the decisions add up to the placed ALLOCs, and spec_rounds grows by the last stage's certification
round of every chunk.  Needs an H100."""
import numpy as np
import pytest

import spec_workloads as SW
from instaslice_b200 import engine as E

pytestmark = pytest.mark.gpu


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _engine(w, flags=0, spec=E.SPEC_AUTO, G=None):
    eng = E.Engine(max_gpus=G or w.G, max_batch=1 << 18, policy=w.policy, quirks=w.quirks, flags=flags)
    eng.set_speculation(spec)
    if w.single_table:
        eng.load_profiles(w.rows)
    else:
        eng.load_profile_tables(w.rows)
    eng.load_inventory(w.node_off, w.occ)
    if w.node_table is not None:
        eng.set_node_tables(w.node_table)
    return eng


def _placed(batches, results):
    return sum(int(np.count_nonzero((b["op"] == E.OP_ALLOC) & (r["status"] == E.ST_PLACED))) for b, r in zip(batches, results))


def _check_trace(tr, before, after, batches, results, n_chunks, what, stages):
    """The invariants of the rounds on the trace [chunk][global stage][12] of one speculative call planned in ``stages`` stages.
    Returns (certification rounds, simulations) [chunk][stage]."""
    assert tr.shape[0] == n_chunks and tr.shape[1] == stages, (what, tr.shape, stages)
    S = stages
    rounds, sims, dec = tr[..., 11].astype(np.int64), tr[..., 7].astype(np.int64), tr[..., 6].astype(np.int64)
    assert after["spec_chunks"] - before["spec_chunks"] == n_chunks, (what, before, after)
    assert (rounds[:, 0] == 1).all(), (what, rounds[:, 0])
    assert (np.diff(rounds, axis=1) >= 0).all(), (what, np.argwhere(np.diff(rounds, axis=1) < 0)[:4])
    assert (rounds >= 1).all() and rounds.max() <= S + 2, (what, int(rounds.max()), S)
    assert (sims <= rounds).all(), (what, np.argwhere(sims > rounds)[:4])
    assert (sims[dec > 0] >= 1).all(), what
    assert int(dec.sum()) == _placed(batches, results), what
    assert after["spec_rounds"] - before["spec_rounds"] == int(rounds[:, -1].sum()), (what, rounds[:, -1])
    return rounds, sims


def _stages(G):
    """The stage count of a single engine's speculative plan: one stage per SM, stage_size GPUs each.  On a 132-SM H100 SXM this is
    the plan the protocol model of test_spec_workloads.py runs."""
    return -(-G // SW.stage_size(G, _sms()))


def _traced_spec_calls(w, wants):
    """Every batch of ``w`` as one traced speculative call; the results are compared and the trace checked.  Returns the engine and the
    (rounds, simulations) of every chunk."""
    eng = _engine(w, E.FLAG_FORCE_PIPELINE | E.FLAG_TRACE, E.SPEC_ON)
    cells = []
    for b, (req, want) in enumerate(zip(w.batches, wants)):
        before = eng.stats()
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (w.name, "spec", b, bad[:4], got[bad[:4]], want[bad[:4]])
        cells.append(_check_trace(eng.read_trace(), before, eng.stats(), [req], [want], _chunks([req]), (w.name, b), _stages(w.G)))
    return eng, cells


def _chunks(batches):
    return sum(-(-len(b) // 65536) for b in batches)


@pytest.mark.parametrize("name", SW.NAMES)
def test_workload_batch_by_batch(name):
    w = SW.build(name)
    wants, final = w.expected()
    eng, _ = _traced_spec_calls(w, wants)
    assert np.array_equal(eng.read_occupancy(), final), (name, "spec")
    eng.close()
    for label, flags, spec in (("plain", E.FLAG_FORCE_PIPELINE, E.SPEC_OFF), ("default", 0, E.SPEC_AUTO)):
        eng = _engine(w, flags, spec)
        for b, (req, want) in enumerate(zip(w.batches, wants)):
            before = eng.stats()
            got = eng.place_batch(req)
            bad = np.flatnonzero(got != want)
            assert len(bad) == 0, (name, label, b, bad[:4], got[bad[:4]], want[bad[:4]])
            if label == "plain":
                assert eng.stats()["spec_chunks"] == before["spec_chunks"], (name, eng.stats())
        assert np.array_equal(eng.read_occupancy(), final), (name, label)
        eng.close()


MULTI = [n for n in SW.NAMES if len(SW.build(n).batches) > 1]


@pytest.mark.parametrize("window", [1, 3])
@pytest.mark.parametrize("name", MULTI)
def test_workload_as_windowed_stream(name, window):
    w = SW.build(name)
    wants, final = w.expected()
    eng = _engine(w, E.FLAG_TRACE, E.SPEC_ON)
    eng.set_causal_window(window)
    before = eng.stats()
    got = eng.place_stream(w.batches)
    for b in range(len(w.batches)):
        assert np.array_equal(got[b], wants[b]), (name, window, b)
    assert np.array_equal(eng.read_occupancy(), final)
    _check_trace(eng.read_trace(), before, eng.stats(), w.batches, wants, _chunks(w.batches), (name, window), _stages(w.G))
    eng.close()


@pytest.mark.parametrize("name", SW.HARDEST)
def test_hardest_workloads_through_an_open_stream(name):
    w = SW.build(name)
    wants, final = w.expected()
    eng = _engine(w, 0, E.SPEC_ON)
    n_total = sum(len(b) for b in w.batches)
    h_in, h_out = E.PinnedArray(n_total, E.REQUEST_DTYPE), E.PinnedArray(n_total, E.RESULT_DTYPE)
    before = eng.stats()
    eng.stream_open(max(2, len(w.batches)))
    off = 0
    for b, req in enumerate(w.batches):
        n = len(req)
        h_in.array[off:off + n] = req
        eng.stream_wait(eng.stream_submit_ptr(n, h_in.ptr + 8 * off, h_out.ptr + 8 * off))
        assert np.array_equal(h_out.array[off:off + n], wants[b]), (name, b)
        off += n
    eng.stream_close()
    assert np.array_equal(eng.read_occupancy(), final)
    after = eng.stats()
    assert after["spec_chunks"] - before["spec_chunks"] == len(w.batches), after
    h_in.free(); h_out.free()
    eng.close()


@pytest.mark.parametrize("n_ranks", [2, 3])
@pytest.mark.parametrize("name", SW.RANK_SUBSET)
def test_workload_across_ranks_on_one_gpu(name, n_ranks):
    """G = 4096 in 64 stages of 64 GPUs over all ranks, as test_gpu_spec.py::test_speculative_rounds_across_ranks_on_one_gpu: the
    engines' stages form one speculative sequence; the owner's result array == the oracle, and the traces of the engines in rank order
    keep the invariants of one sequence."""
    import torch
    from instaslice_b200 import dist as D
    w = SW.build(name, 4096)
    wants, final = w.expected()
    sizes = np.array([len(b) for b in w.batches], dtype=np.uint32)
    n_ops = int(sizes.sum())
    d_in = torch.from_numpy(np.concatenate(w.batches).view(np.int64).copy()).cuda()
    bounds = D.all_bounds(w.G, n_ranks, align=64)
    cuts = [lo for lo, _ in bounds] + [w.G]
    engines = []
    for lo, hi in bounds:
        eng = _engine(w, E.FLAG_TRACE)
        eng.ipc_inbox_handle(); eng.ipc_spec_handle()
        engines.append(eng)
    for r, eng in enumerate(engines):
        eng.connect_local(engines[r + 1] if r + 1 < n_ranks else None, has_prev=r > 0)
        eng.connect_owner_local(engines[0] if r > 0 else None)
        eng.set_ring_world(n_ranks)
        eng.connect_spec_local(n_ranks, r, engines, cuts)
        eng.set_causal_window(1)
        eng.set_speculation(E.SPEC_ON)
    torch.cuda.synchronize()
    for eng, (lo, hi) in zip(engines, bounds):
        eng.set_partition(lo, hi)
    before = [eng.stats() for eng in engines]
    for eng in engines:
        eng.place_stream_partitioned(sizes, d_in.data_ptr(), eng.device_results(), 1)
    for eng in engines:
        eng.synchronize()

    class _View:            # torch view of the owner's engine-owned result array (no copy)
        __cuda_array_interface__ = {"shape": (n_ops,), "typestr": "<i8", "data": (engines[0].device_results(), False), "version": 3}
    got = torch.as_tensor(_View(), device="cuda").cpu().numpy().view(E.RESULT_DTYPE)
    assert np.array_equal(got, np.concatenate(wants)), (name, n_ranks)
    occ = np.concatenate([eng.read_occupancy()[lo:hi] for eng, (lo, hi) in zip(engines, bounds)])
    assert np.array_equal(occ, final)
    after = [eng.stats() for eng in engines]
    tr = np.concatenate([eng.read_trace() for eng in engines], axis=1)
    # 64 stages of 64 GPUs over all ranks; the last rank's engine counts the rounds and chunks of the sequence
    _check_trace(tr, before[-1], after[-1], w.batches, wants, _chunks(w.batches), (name, n_ranks), 64)
    for eng in engines:
        eng.close()


@pytest.mark.parametrize("name", ["order_big_first", "skew_1g_2g", "size1_only"])
def test_rounds_take_both_branches_of_the_simulation(name):
    """On each of these workloads some cell is simulated more than once (its entry was corrected) and some cell is certified with fewer
    simulations than rounds (an unchanged entry is not simulated again)."""
    w = SW.build(name)
    wants, _ = w.expected()
    eng, cells = _traced_spec_calls(w, wants)
    eng.close()
    assert any((sims >= 2).any() for _, sims in cells), name
    assert any((sims < rounds).any() for rounds, sims in cells), name
