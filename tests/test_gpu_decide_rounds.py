"""The decision loop of k_pipeline is a latency-tuned restatement of one recurrence: however it is scheduled, every simulation of a
stage must log the same decisions, so the speculative rounds certify every stage in the same round.  This file holds the device to that
on every table of golden/tables.json under both quirk sets and on every workload of spec_workloads.py: results and final occupancy
against ``oracle.Fast`` byte for byte, and the certification round of every (chunk, stage) cell (trace word 11) against
golden/decide_rounds.json, recorded on an H100 SXM (132 SMs) from the loop that logged every decision as it was made.

Regenerate the golden file (on a 132-SM H100, from a build whose rounds are known to be right):
    python tests/test_gpu_decide_rounds.py --write
Needs an H100."""
import json
import os
import sys

import numpy as np
import pytest

for _p in (os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__)))):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import oracle  # noqa: E402
import spec_workloads as SW  # noqa: E402
from instaslice_b200 import engine as E, tables, workloads as W  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decide_rounds.json")
TABLE_CASES = [(t, q) for t in sorted(tables.TABLES) for q in (E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED)]


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _table_workload(tname, quirks):
    """Two batches on 8192 GPUs of random occupancy: uniform profiles of the table, then FREEs of half the first batch's placements
    with a second uniform batch (the oracle's placements, so that the FREEs are valid)."""
    rows = E.make_profiles(tables.TABLES[tname])
    rng = W.SplitMix64(101 + 7 * quirks + len(tname))
    node_off = W.node_offsets(1024, 8)
    occ = (rng.next(8192) & np.uint64(0x3F)).astype(np.uint8)
    n_prof = len(rows)
    first = W.alloc_requests((rng.next(60000) % np.uint64(n_prof)).astype(np.uint8))
    ref = oracle.Fast(node_off, rows, quirks)
    ref.load(occ)
    placed = ref.place(first)
    live = placed[placed["status"] == E.ST_PLACED][::2]
    frees = np.zeros(len(live), dtype=E.REQUEST_DTYPE)
    frees["handle"], frees["op"], frees["start"], frees["size"] = live["gpu"], E.OP_FREE, live["start"], live["size"]
    second = np.concatenate([frees, W.alloc_requests((rng.next(40000) % np.uint64(n_prof)).astype(np.uint8))])
    return rows, node_off, occ, [first, second]


def _spec_calls(rows, node_off, occ, batches, quirks, policy=E.POLICY_FIRST_FIT, node_table=None, single_table=True):
    """Every batch as one traced speculative call, checked against the oracle; returns per call the certification round of every
    (chunk, stage) cell."""
    ref = oracle.Fast(node_off, rows, quirks, policy=policy, node_table=node_table)
    ref.load(occ)
    eng = E.Engine(max_gpus=int(node_off[-1]), max_batch=1 << 18, policy=policy, quirks=quirks, flags=E.FLAG_FORCE_PIPELINE | E.FLAG_TRACE)
    eng.set_speculation(E.SPEC_ON)
    if single_table:
        eng.load_profiles(rows)
    else:
        eng.load_profile_tables(rows)
    eng.load_inventory(node_off, occ)
    if node_table is not None:
        eng.set_node_tables(node_table)
    calls = []
    for b, req in enumerate(batches):
        want = ref.place(req)
        got = eng.place_batch(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (b, bad[:4], got[bad[:4]], want[bad[:4]])
        calls.append(eng.read_trace()[..., 11].astype(np.int64).tolist())
    assert np.array_equal(eng.read_occupancy(), ref.occupancy())
    eng.close()
    return calls


def table_case(tname, quirks):
    rows, node_off, occ, batches = _table_workload(tname, quirks)
    return _spec_calls(rows, node_off, occ, batches, quirks)


def workload_case(name):
    w = SW.build(name)
    return _spec_calls(w.rows, w.node_off, w.occ, w.batches, w.quirks, w.policy, w.node_table, w.single_table)


def _golden():
    with open(GOLDEN) as f:
        g = json.load(f)
    if _sms() != g["sms"]:
        pytest.skip("golden rounds were recorded on a %d-SM GPU; the stage plan differs on %d SMs" % (g["sms"], _sms()))
    return g


def _check(got, want, what):
    assert len(got) == len(want), what
    for b, (g, w) in enumerate(zip(got, want)):
        g, w = np.array(g), np.array(w)
        assert g.shape == w.shape, (what, b, g.shape, w.shape)
        bad = np.argwhere(g != w)
        assert len(bad) == 0, (what, b, "cells (chunk, stage) certified in another round", bad[:4].tolist(), g[tuple(bad[0])], w[tuple(bad[0])])


@pytest.mark.parametrize("tname,quirks", TABLE_CASES)
def test_table_rounds_match_golden(tname, quirks):
    _check(table_case(tname, quirks), _golden()["tables"]["%s/%d" % (tname, quirks)], (tname, quirks))


@pytest.mark.parametrize("name", SW.NAMES)
def test_workload_rounds_match_golden(name):
    _check(workload_case(name), _golden()["workloads"][name], name)


if __name__ == "__main__":
    if "--write" not in sys.argv:
        sys.exit(__doc__)
    out = {"sms": _sms(), "gpu": __import__("torch").cuda.get_device_name(0),
           "tables": {"%s/%d" % (t, q): table_case(t, q) for t, q in TABLE_CASES},
           "workloads": {n: workload_case(n) for n in SW.NAMES}}
    with open(sys.argv[sys.argv.index("--write") + 1] if len(sys.argv) > sys.argv.index("--write") + 1 else GOLDEN, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
