"""The structured workloads of spec_workloads.py on the CPU: the two oracles agree on them, the protocol model of the speculative rounds
(spec_rounds_model.cpp --world) is sound, makes progress and terminates within stages + 2 rounds on every single-table workload, bounded
and unbounded, and every workload not marked as an edge shape costs the model more rounds than every one of its baselines — the same
requests shuffled, or the same occupancy bytes permuted, at the same stage size, with each of twelve seeds."""
import os
import subprocess

import numpy as np
import pytest

import oracle
import spec_workloads as SW
from instaslice_b200 import engine as E

SINGLE = [n for n in SW.NAMES if SW.build(n).single_table]


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    return SW.build_model(str(tmp_path_factory.mktemp("model") / "spec_rounds_model"))


def _rounds(model, tmp_path, worlds, bounded=False):
    out = []
    for w in worlds:
        rc, text, rounds = SW.run_model(model, w, str(tmp_path), bounded)
        assert rc == 0 and rounds is not None, text
        out.append(rounds)
    return out


def test_stage_size_matches_the_plan_for_132_sms():
    """segment_geometry's speculative branch: target = SMs, sub = max(64, ceil(G / SMs)) rounded up to 64 — the arithmetic
    test_gpu_table_limits.py::test_plan_boundaries_for_128_candidates pins on the device (SMs x 64 GPUs is the last one-stage-per-SM
    inventory of 64-GPU stages)."""
    assert SW.stage_size(132 * 64) == 64 and SW.stage_size(132 * 64 + 64) == 128
    assert SW.stage_size(4096) == 64 and SW.stage_size(8192) == 64 and SW.stage_size(16384) == 128
    for name in SW.NAMES:
        w = SW.build(name)
        S = -(-w.G // SW.stage_size(w.G))
        assert 2 <= S <= 132, (name, S)          # one stage per SM: the speculative plan exists


@pytest.mark.parametrize("name", SW.NAMES)
def test_workload_is_well_formed(name):
    """FREEs name spans that are live when their batch starts; the workload is adversarial or says why it is an edge shape."""
    w = SW.build(name)
    assert (w.baseline in ("shuffle", "permute")) != bool(w.edge), name
    results, _ = w.expected()
    for req, res in zip(w.batches, results):
        assert (res["status"][req["op"] == E.OP_FREE] == E.ST_FREED).all()
        assert len(req) <= (1 << 18)


def test_workloads_reach_their_edges():
    full = SW.build("exactly_full")
    (res,), occ = full.expected()
    assert (res["status"] == E.ST_PLACED).all() and (occ & 0x7F == 0x7F).all()
    dry = SW.build("dry_at_stage_boundary")
    (res,), _ = dry.expected()
    sub = SW.stage_size(dry.G)
    req = dry.batches[0]
    g4 = res["gpu"][req["profile"] == SW.P4G]
    assert (res["status"][req["profile"] == SW.P4G] == E.ST_PLACED).all()
    last = int(g4.max())
    assert last // sub != int(g4.min()) // sub                            # the queue lasts over several stages ...
    assert (req["profile"][np.flatnonzero(req["profile"] == SW.P4G)[-1] + 1:] != SW.P4G).all()
    tail = SW.build("free_heavy_tail")
    cut = tail.G - 8 * SW.stage_size(tail.G)
    for req in tail.batches[1:]:
        frees = req[req["op"] == E.OP_FREE]
        assert len(frees) > 0 and (frees["handle"] >= cut).all()
    (res,), occ = SW.build("nothing_placeable").expected()
    assert (res["status"] == E.ST_NO_CAPACITY).all()
    assert SW.build("chunks_131077").batches[0].size > 2 * 65536


@pytest.mark.parametrize("name", SW.NAMES)
def test_fast_equals_faithful_on_a_small_instance(name):
    """The first 512 GPUs (whole nodes) and the first 1500 ALLOCs of every batch, FREEs dropped: the reference as written (slow, so
    small) against the bitmask oracle every device test checks with.  First fit: ref_faithful has no other policy."""
    w = SW.build(name)
    n_nodes = int(np.searchsorted(w.node_off, min(w.G, 512), side="right")) - 1
    node_off = w.node_off[:n_nodes + 1]
    G = int(node_off[-1])
    nt = None if w.node_table is None else w.node_table[:n_nodes]
    fast = oracle.Fast(node_off, w.rows, w.quirks, 0, nt)
    fast.load(w.occ[:G])
    slow = oracle.Faithful(node_off, w.rows, w.quirks, nt)
    slow.load_occupancy_as_dangling(w.occ[:G])
    for b, req in enumerate(w.batches):
        allocs = req[req["op"] == E.OP_ALLOC][:1500]
        a, f = slow.place(allocs), fast.place(allocs)
        assert np.array_equal(a, f), (name, b, int(np.argmax(a != f)))
        assert np.array_equal(slow.occupancy(), fast.occupancy()), (name, b)


@pytest.mark.parametrize("name", SINGLE)
def test_model_is_sound_and_terminates(name, model, tmp_path):
    """Soundness, progress, no move of a consistent prefix and termination within stages + 2 rounds, with the simulations unbounded and
    bounded; an adversarial workload costs more rounds than the most its seeded baselines take."""
    w = SW.build(name)
    worlds = SW.worlds(w)
    S = -(-w.G // SW.stage_size(w.G))
    free = _rounds(model, tmp_path, worlds)
    bounded = _rounds(model, tmp_path, worlds, bounded=True)
    assert max(free + bounded) <= S + 2
    if w.baseline:
        base = [sum(_rounds(model, tmp_path, [x.shuffled(seed) if w.baseline == "shuffle" else x.permuted(seed) for x in worlds]))
                for seed in SW.BASELINE_SEEDS]
        assert sum(free) > max(base), (name, free, base)


def test_hardest_workloads_are_the_hardest(model, tmp_path):
    """The open-stream device test runs the four workloads with the most model rounds whose batches fit one stream slot."""
    rounds = {}
    for name in SINGLE:
        w = SW.build(name)
        if max(len(b) for b in w.batches) <= 65536:
            rounds[name] = max(_rounds(model, tmp_path, SW.worlds(w)))
    assert set(SW.HARDEST) <= set(rounds) and len(SW.HARDEST) == 4
    assert min(rounds[n] for n in SW.HARDEST) >= max(r for n, r in rounds.items() if n not in SW.HARDEST), rounds


def test_model_notices_a_certification_without_the_consistency_of_the_stage_itself(tmp_path):
    """Certifying a stage on the bits of the stages in front alone (dropping c(s, r-1)) certifies entries that are not the true token:
    the model fails on the structured workloads.  The mutant is compiled from the model's source with the one term removed."""
    src = open(os.path.join(SW.ROOT, "tests", "spec_rounds_model.cpp")).read()
    assert src.count("if (allc && cprev[s]) {") == 1
    mutant = tmp_path / "mutant.cpp"
    mutant.write_text(src.replace("if (allc && cprev[s]) {", "if (allc) {"))
    exe = str(tmp_path / "mutant")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, str(mutant)], check=True)
    for name in ("order_big_first", "size1_only"):
        (world,) = SW.worlds(SW.build(name))          # one chunk
        rc, text, _ = SW.run_model(exe, world, str(tmp_path), False)
        assert rc != 0 and "FAIL: unsound certification" in text, (name, text)
