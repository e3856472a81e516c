"""The per-(chunk, stage) trace of the segment pipeline (FLAG_TRACE, ``Engine.read_trace``): every cell records the decisions it
committed and globaltimer stamps of its steps.  The decisions of all cells must add up to what was placed, and the stamps of a cell
that placed anything must follow the order of the pipeline's steps.  Up to 16 384 GPUs every stage is one sub-segment, so no stamp of
a cell is overwritten by a later sub-segment.  Needs an H100."""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables, workloads as W

pytestmark = pytest.mark.gpu

G = 8192
# trace words (isl_read_trace): 0 cell start (rounds: sweep + prediction done), 1 token in, 2 token out (rounds: certified),
# 3 commit done, 4 chain start, 5 chain end, 6 decisions, 8 heads done, 9 windows staged, 11 rounds (speculative pipeline)
PLAIN_ORDER = (1, 8, 9, 4, 5, 2, 3)
IDLE_ORDER = (1, 8, 2, 3)           # a stage with nothing pending passes the token on at once: token out == commit done
SPEC_ORDER = (0, 2, 3)


def _setup(seed):
    rows = E.make_profiles(tables.H100_80GB)
    rng = W.SplitMix64(seed)
    node_off = W.node_offsets(G // 8, 8)
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    ref = oracle.Fast(node_off, rows)
    ref.load(occ)
    return rows, rng, node_off, occ, ref


def _engine(rows, node_off, occ, mode):
    eng = E.Engine(max_gpus=G, max_batch=1 << 18, flags=E.FLAG_TRACE | E.FLAG_FORCE_PIPELINE)
    eng.set_speculation(mode)
    eng.load_profiles(rows)
    eng.load_inventory(node_off, occ)
    return eng


def _placed(batches, results):
    return sum(int(np.count_nonzero((b["op"] == E.OP_ALLOC) & (r["status"] == E.ST_PLACED))) for b, r in zip(batches, results))


def _check_order(tr, order):
    busy = tr[..., 6] > 0
    assert busy.any()
    stamps = tr[busy][:, list(order)]
    assert (stamps > 0).all()
    bad = np.flatnonzero((np.diff(stamps.astype(np.int64), axis=1) < 0).any(axis=1))
    assert len(bad) == 0, stamps[bad[:4]]
    return busy


def test_plain_pipeline_trace():
    rows, rng, node_off, occ, ref = _setup(2024)
    first = W.alloc_requests(W.mix_profiles(rng, 4000))
    want_first = ref.place(first)
    live = want_first[want_first["status"] == E.ST_PLACED][:3000]
    frees = np.zeros(len(live), dtype=E.REQUEST_DTYPE)
    frees["handle"], frees["op"], frees["start"], frees["size"] = live["gpu"], E.OP_FREE, live["start"], live["size"]
    # the first batch is placed by the first few stages: the stages behind them pass the token on (idle cells)
    stream = [W.alloc_requests(W.mix_profiles(rng, 300)), np.concatenate([frees[:1500], W.alloc_requests(W.mix_profiles(rng, 6000))]),
              np.concatenate([frees[1500:], W.alloc_requests(W.mix_profiles(rng, 30000))])]
    want = [ref.place(b) for b in stream]
    eng = _engine(rows, node_off, occ, E.SPEC_OFF)
    assert np.array_equal(eng.place_batch(first), want_first)
    steps = eng.stats()["chain_steps"]
    got = eng.place_stream(stream)
    for b in range(len(stream)):
        assert np.array_equal(got[b], want[b]), b
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    st = eng.stats()
    tr = eng.read_trace()
    assert tr.shape[0] == len(stream) and tr.shape[1] > 1
    placed = _placed(stream, want)
    assert placed > 0
    assert int(tr[..., 6].sum()) == st["chain_steps"] - steps == placed
    _check_order(tr, PLAIN_ORDER)
    idle = (tr[..., 6] == 0) & (tr[..., 2] > 0) & (tr[..., 2] == tr[..., 3])
    assert idle[0].any()
    stamps = tr[idle][:, list(IDLE_ORDER)].astype(np.int64)
    assert (stamps > 0).all() and (np.diff(stamps, axis=1) >= 0).all()
    assert st["spec_chunks"] == 0, st
    eng.close()


def test_speculative_pipeline_trace():
    rows, rng, node_off, occ, ref = _setup(4048)
    req = W.alloc_requests(W.mix_profiles(rng, 40000))
    want = ref.place(req)
    eng = _engine(rows, node_off, occ, E.SPEC_ON)
    got = eng.place_batch(req)
    assert np.array_equal(got, want), int(np.argmax(got != want))
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    st = eng.stats()
    assert st["spec_chunks"] == 1 and st["spec_rounds"] >= 1, st
    tr = eng.read_trace()
    assert tr.shape[0] == 1 and tr.shape[1] > 1
    assert int(tr[..., 6].sum()) == _placed([req], [want]) > 0
    busy = _check_order(tr, SPEC_ORDER)
    assert (tr[busy][:, 11] >= 1).all()
    eng.close()
