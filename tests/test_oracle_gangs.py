"""All-or-nothing gangs (isl_place_gangs) on the CPU: the hand-derived known-answer vector, the two restatements of tests/gang_oracle.py
against each other, and the C ABI's argument checks that need no device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200.workloads import SplitMix64, alloc_requests, node_offsets

import gang_oracle as GO
from gang_oracle import A100, KAT_GANGS, KAT_OCC, KAT_RECORDS, kat_call

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ST_N = E.ST_NO_CAPACITY


def test_kat_fast():
    rows = E.make_profiles(tables.A100_40GB)
    req, off = kat_call()
    # gang by gang, so that the occupancy after each one is seen; then all gangs in one call
    ref = oracle.Fast(node_offsets(1, 1), rows, 3, 0)
    ref.load(np.zeros(1, dtype=np.uint8))
    for i, (a, b) in enumerate(zip(off[:-1], off[1:])):
        got = GO.fast_place_gangs(ref, req[a:b], [0, b - a], GO.default_sizes(rows))
        assert [tuple(int(x) for x in r) for r in got] == KAT_RECORDS[i], i
        assert int(ref.occupancy()[0]) == KAT_OCC[i], i
    ref.load(np.zeros(1, dtype=np.uint8))
    got = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows))
    assert [tuple(int(x) for x in r) for r in got] == [r for g in KAT_RECORDS for r in g]
    assert int(ref.occupancy()[0]) == KAT_OCC[-1]


def test_kat_ref_py():
    crs = GO.cluster_crs([0, 1], [0], [0], [tables.A100_40GB])
    k = iter(range(100))
    for i, gang in enumerate(KAT_GANGS):
        pods = [({"uid": "u%d" % next(k), "name": "p"}, name) for name in gang]
        (verdict, detail), = GO.ref_py_place_gangs(crs, [pods], 3)
        placed = [r for r in KAT_RECORDS[i] if r[3] == E.ST_PLACED]
        if placed:
            assert verdict == "placed" and [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in detail] == [r[:3] for r in placed], i
        else:
            failed = next(j for j, r in enumerate(KAT_RECORDS[i]) if r[3] == ST_N)
            assert (verdict, detail) == ("aborted", failed), i
        assert int(GO.cr_occupancy(crs)[0]) == KAT_OCC[i], i


def test_gang_spans_nodes_fast():
    """Two nodes of one GPU each: the gang [3g.20gb, 3g.20gb] is placed on GPU 0 and GPU 1."""
    rows = E.make_profiles(tables.A100_40GB)
    ref = oracle.Fast(node_offsets(2, 1), rows, 3, 0)
    ref.load(np.zeros(2, dtype=np.uint8))
    got = GO.fast_place_gangs(ref, alloc_requests(np.array([A100["3g.20gb"]] * 2, dtype=np.uint8)), [0, 2], GO.default_sizes(rows))
    assert [tuple(int(x) for x in r) for r in got] == [(0, 0, 4, E.ST_PLACED), (1, 0, 4, E.ST_PLACED)]


def random_gangs(rng, n, max_size):
    """Gang offsets of a random partition of n requests into gangs of 1..max_size."""
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % max_size)))
    return np.asarray(off, dtype=np.uint32)


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
@pytest.mark.parametrize("hetero", [False, True])
def test_fast_and_ref_py_agree(quirks, hetero):
    """Random CR states and random gang partitions, first-fit: the two restatements give the same records and occupancy."""
    rng = SplitMix64(1000 + quirks * 2 + hetero)
    tabs = [tables.A100_40GB, tables.H100_80GB] if hetero else [tables.H100_80GB]
    names, rows2d = E.make_profile_tables(tabs)
    for trial in range(4):
        n_nodes = 2 + int(rng.next1() % 4)
        node_table = (rng.next(n_nodes) % np.uint64(len(tabs))).astype(np.uint8)
        node_off = np.concatenate([[0], np.cumsum(1 + (rng.next(n_nodes) % np.uint64(3)).astype(np.int64))]).astype(np.uint32)
        G = int(node_off[-1])
        occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
        n = 20 + int(rng.next1() % 40)
        prof = (rng.next(n) % np.uint64(len(names))).astype(np.uint8)
        req = alloc_requests(prof)
        off = random_gangs(rng, n, 5)
        ref = oracle.Fast(node_off, rows2d, quirks, 0, node_table=node_table)
        ref.load(occ)
        got = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows2d, node_table))
        crs = GO.cluster_crs(node_off, node_table, occ, tabs)
        gangs = [[({"uid": "u%d" % i, "name": "p%d" % i}, names[prof[i]]) for i in range(a, b)] for a, b in zip(off[:-1], off[1:])]
        want = GO.ref_py_place_gangs(crs, gangs, quirks)
        for gi, ((a, b), (verdict, detail)) in enumerate(zip(zip(off[:-1], off[1:]), want)):
            recs = got[a:b]
            if verdict == "placed":
                assert (recs["status"] == E.ST_PLACED).all(), (trial, gi)
                assert [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in recs] == \
                       [(int(x["gpuUUID"][4:]), x["start"], x["size"]) for x in detail], (trial, gi)
            else:
                assert recs["status"][detail] == E.ST_NO_CAPACITY, (trial, gi)
                assert (np.delete(recs["status"], detail) == E.ST_GANG_ABORTED).all(), (trial, gi)
        assert np.array_equal(ref.occupancy(), GO.cr_occupancy(crs)), trial


@pytest.mark.parametrize("policy", [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG])
def test_gangs_of_one_equal_place(policy):
    """A call whose gangs all have one member is the batch call: same records, same occupancy (FREEs and NOOPs included)."""
    rng = SplitMix64(40 + policy)
    rows = E.make_profiles(tables.H100_80GB)
    node_off = node_offsets(8, 4)
    G = int(node_off[-1])
    occ = ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)
    req = alloc_requests((rng.next(200) % np.uint64(len(rows) + 1)).astype(np.uint8))
    req["profile"][req["profile"] == len(rows)] = E.PROFILE_UNKNOWN
    for i in range(0, 200, 17):
        g = int(rng.next1() % G)
        req[i] = (g, 0, E.OP_FREE, 0, 1 + int(rng.next1() % 2))
    req["op"][5::23] = E.OP_NOOP
    a = oracle.Fast(node_off, rows, 3, policy)
    a.load(occ)
    b = oracle.Fast(node_off, rows, 3, policy)
    b.load(occ)
    got = GO.fast_place_gangs(a, req, np.arange(len(req) + 1, dtype=np.uint32), GO.default_sizes(rows))
    assert np.array_equal(got, b.place(req))
    assert np.array_equal(a.occupancy(), b.occupancy())


def test_dropping_an_aborted_gang_changes_nothing_else():
    rng = SplitMix64(5)
    rows = E.make_profiles(tables.A100_40GB)
    node_off = node_offsets(4, 2)
    G = int(node_off[-1])
    occ = (rng.next(G) & np.uint64(0x33)).astype(np.uint8)
    req = alloc_requests((rng.next(60) % np.uint64(len(rows))).astype(np.uint8))
    off = random_gangs(rng, len(req), 6)
    sizes = GO.default_sizes(rows)
    ref = oracle.Fast(node_off, rows, 3, 0)
    ref.load(occ)
    full = GO.fast_place_gangs(ref, req, off, sizes)
    final = ref.occupancy()
    aborted = [k for k, (a, b) in enumerate(zip(off[:-1], off[1:])) if (full["status"][a:b] == E.ST_GANG_ABORTED).any()]
    assert aborted, "the vector must contain an aborted gang"
    for k in aborted:
        a, b = int(off[k]), int(off[k + 1])
        keep = np.r_[0:a, b:len(req)]
        off2 = np.concatenate([off[:k + 1], off[k + 2:] - (b - a)]).astype(np.uint32)
        ref.load(occ)
        got = GO.fast_place_gangs(ref, req[keep], off2, sizes)
        assert np.array_equal(got, full[keep]), k
        assert np.array_equal(ref.occupancy(), final), k


def test_place_gangs_argument_validation_without_gpu():
    """The checks that need no engine return ISL_EINVAL before any CUDA call."""
    lib = E.load_library()
    req = alloc_requests(np.zeros(2, dtype=np.uint8))
    out = np.zeros(2, dtype=E.RESULT_DTYPE)
    off = np.array([0, 2], dtype=np.uint32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert lib.isl_place_gangs(None, 1, p(off), p(req), p(out)) == E.EINVAL
    assert lib.isl_place_gangs(None, 0, None, None, None) == E.EINVAL


def test_place_gangs_header_is_plain_c99(tmp_path):
    if not shutil.which("gcc"):
        pytest.skip("no gcc")
    src = tmp_path / "t.c"
    src.write_text('#include "islplace.h"\n'
                   'int f(isl_engine* e) { uint32_t off[2] = {0, 1}; isl_request r = {0, 0, ISL_OP_ALLOC, 0, 0}; isl_result s;\n'
                   '  return isl_place_gangs(e, 1, off, &r, &s) == ISL_OK && s.status == ISL_ST_GANG_ABORTED; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(tmp_path / "t.o")], check=True)
