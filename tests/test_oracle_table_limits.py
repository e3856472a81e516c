"""Profile tables at the limits the ABI accepts (include/islplace.h): 16 profile names, 8 node tables, 8 starts per row and 128
(table, profile, start) candidates — and the CPU pins of the oracle on them (CPU only).

The fixtures are built here, deterministically from seeded splitmix64, and ``test_gpu_table_limits.py`` runs the same ones through every
device path.  The self-checks below make sure each fixture really reaches the edge it exists for, so that the device tests cannot pass
by missing it:
  T16x8      16 size-1 rows, each with all 8 starts in its own order: 128 candidates under every quirk set (K = 4 lane slots), and
             profile 15 in use, which selects the P15 form of the pipeline's decision loop
  T16mix-1/2 16 rows of sizes 1..8, unordered starts, starts with start + size > 8, one row (index 15) no quirk set can place:
             <= 32 candidates (K = 1) / 33..64 candidates (K = 2) under every quirk set
  T8tab      8 tables over 16 names, each table knowing a sparse subset; profile 15 known to table 7 only, which is not the table of
             node 0; exactly 128 candidates under FIXED quirks, more than 32 of them 4 slices or wider; one more candidate is rejected
  T16top     15 size-1 rows of 8 starts and one size-8 row: the largest ISL_POLICY_MIN_FRAG score a table can produce (121)
  Edge65535  T16x8 on a few thousand GPUs, one chunk of exactly 65 536 requests whose last one (in-chunk index 65535, key
             t << 15 | p << 11 with every bit of 11..30 set) is profile 15 and is placed while other profiles' queues are exhausted
"""
import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

QUIRK_SETS = (0, 1, 2, 3)
EDGE_N = 65536
EDGE_G = 4096


# ---- a restatement of candidate_mask (isl_kernels.cuh) and what follows from it ----------------------------------------------------
def candidate_mask(size, v, quirks):
    """Slot mask of placing a ``size``-slice profile at start ``v``, or 0 when the search can never return ``v``."""
    size, v = int(size), int(v)
    if v >= 8 or size == 0 or size > 8:
        return 0
    if size == 1:
        return 1 << v
    if quirks & E.QUIRK_POW2_ONLY and size not in (2, 4, 8):
        return 0
    if (v + size >= 8) if quirks & E.QUIRK_STRICT_BOUND else (v + size > 8):
        return 0
    return (((1 << size) - 1) << v) & 0xFF


def candidates(rows, quirks):
    """(table, profile, start, mask) of every candidate of [P] or [T][P] rows, in the engine's order."""
    rows2 = rows if rows.ndim == 2 else rows[None]
    out = []
    for t in range(rows2.shape[0]):
        for p in range(rows2.shape[1]):
            row = rows2[t, p]
            for k in range(int(row["n_starts"])):
                m = candidate_mask(row["size"], row["starts"][k], quirks)
                if m:
                    out.append((t, p, int(row["starts"][k]), m))
    return out


def cand_slots(n):
    """K of k_chain<K> / k_small<K> / k_pipeline<K, ..> for n candidates."""
    return 1 if n <= 32 else (2 if n <= 64 else 4)


def min_frag_scores(rows, quirks):
    """[profile][occupancy byte] -> (profile, start) pairs of the table that stop being feasible when the profile takes its first legal
    start there (what ISL_POLICY_MIN_FRAG minimises); 0 where the profile has no legal start."""
    masks = [m for _, _, _, m in candidates(rows, quirks)]
    score = np.zeros((len(rows), 256), dtype=np.int64)
    for p in range(len(rows)):
        for o in range(256):
            mine = next((m for m in (candidate_mask(rows[p]["size"], s, quirks) for s in rows[p]["starts"][:rows[p]["n_starts"]])
                         if m and o & m == 0), 0)
            if mine:
                score[p, o] = sum(1 for m in masks if o & m == 0 and (o | mine) & m)
    return score


# ---- fixtures ------------------------------------------------------------------------------------------------------------------------
def t16x8():
    """16 size-1 rows: rows 0..7 the rotations of 0..7, rows 8..15 the reversed rotations."""
    table = [("x%d" % i, 1, [(j + i) % 8 for j in range(8)] if i < 8 else [(i - j) % 8 for j in range(8)], i) for i in range(16)]
    return E.make_profiles(table)


# (size, starts) per row; T16mix-1 keeps the first start of every row except rows 0 and 15, T16mix-2 keeps them all
_MIX = [
    (1, [3, 0, 7, 5, 1, 6, 2, 4]),      # 8 starts: order 7
    (2, [6, 0, 4, 2, 5, 7, 1, 3]),      # 6 + 2 = 8: FIXED only; 7 + 2 > 8: never
    (3, [5, 0, 2]),
    (4, [4, 0, 2, 3, 1, 6]),
    (5, [3, 1, 0, 2, 5]),
    (6, [2, 0, 1, 4]),
    (7, [1, 0, 3]),
    (8, [0, 2]),
    (1, [7, 6, 5, 4, 0, 2]),
    (2, [2, 4, 0, 6, 1, 3, 5]),
    (4, [0, 4, 2, 1, 5]),
    (3, [4, 1, 5]),
    (6, [0, 2, 1]),
    (5, [2, 0, 3, 1]),
    (2, [7, 1, 3, 5, 0]),
    (3, [7, 6]),                        # size 3 at 6 or 7: no quirk set places it
]


def t16mix(variant):
    assert variant in (1, 2)
    return E.make_profiles([("m%d" % i, size, starts if variant == 2 or i in (0, 15) else starts[:1], i)
                            for i, (size, starts) in enumerate(_MIX)])


def t16top():
    """15 size-1 rows of 8 starts and a size-8 row (index 15): a size-8 placement on an empty GPU kills all 121 pairs (FIXED quirks)."""
    return E.make_profiles([("x%d" % i, 1, [(j + i) % 8 for j in range(8)], i) for i in range(15)] + [("full", 8, [0], 15)])


def t8tab(budget=128):
    """[8][16] rows.  Every table knows about two thirds of the names (n_starts == 0 elsewhere), profile 15 only table 7; sizes lean to
    4..8 slices.  Starts are handed out one round at a time over all rows, so that every table gets its share, until ``budget``
    candidates under FIXED quirks; illegal starts ride along."""
    rng = W.SplitMix64(8008)
    sizes = (1, 2, 3, 4, 4, 5, 5, 6, 6, 7, 8, 8)
    plan = []
    for t in range(8):
        for p in range(16):
            if (p == 15 and t != 7) or (p != 15 and rng.next1() % 3 == 0):
                continue
            plan.append((t, p, sizes[rng.next1() % len(sizes)], [int(s) for s in np.argsort(rng.next(8), kind="stable")]))
    rows = np.zeros((8, 16), dtype=E.PROFILE_DTYPE)
    total = 0
    for r in range(8):
        for t, p, size, perm in plan:
            if total == budget:
                break
            n = int(rows["n_starts"][t, p])
            rows["size"][t, p] = size
            rows["starts"][t, p, n] = perm[r]
            rows["n_starts"][t, p] = n + 1
            rows["gi"][t, p] = rows["ci"][t, p] = p
            total += candidate_mask(size, perm[r], E.QUIRKS_FIXED) != 0
    return rows


def plus_one_candidate(rows, quirks):
    """A copy of ``rows`` with one more legal start in the first row that has room for one."""
    rows = rows.copy()
    rows2 = rows if rows.ndim == 2 else rows[None]
    for t, p in np.ndindex(rows2.shape):
        n = int(rows2["n_starts"][t, p])
        if 0 < n < 8:
            used = set(int(s) for s in rows2["starts"][t, p, :n])
            for s in range(8):
                if s not in used and candidate_mask(rows2["size"][t, p], s, quirks):
                    rows2["starts"][t, p, n] = s
                    rows2["n_starts"][t, p] = n + 1
                    return rows
    raise AssertionError("no row has room for another candidate")


def ragged_nodes(rng, n_nodes, max_gpus=8):
    return np.concatenate([[0], np.cumsum(1 + (rng.next(n_nodes) % np.uint64(max_gpus)).astype(np.int64))]).astype(np.uint32)


def t8tab_node_tables(rng, n_nodes):
    """Table of every node: random, node 0 on table 2 (a table that does not know every name), table 7 first seen later."""
    node_table = (rng.next(n_nodes) % np.uint64(8)).astype(np.uint8)
    node_table[:3] = (2, 0, 5)[:n_nodes]
    return node_table


def edge65535(rng):
    """(node_off, occ, requests) of Edge65535 on T16x8: 4096 GPUs about one eighth busy; one chunk of 65 536 requests, about a third
    of them ALLOCs (the rest NOOPs and unknown profiles) so that every ALLOC fits; profile 3 only among the first 1024 requests; the
    last request is profile 15."""
    node_off = W.node_offsets(EDGE_G // 8, 8)
    occ = (rng.next(EDGE_G) & rng.next(EDGE_G) & rng.next(EDGE_G) & np.uint64(0xFF)).astype(np.uint8)
    return node_off, occ, edge_requests(rng, EDGE_N)


def edge_requests(rng, n):
    req = W.alloc_requests((rng.next(n) % np.uint64(16)).astype(np.uint8))
    kind = rng.next(n) % np.uint64(8)
    late3 = (req["profile"] == 3) & (np.arange(n) >= 1024)
    req["profile"][late3] = 4
    req["op"][kind >= 3] = E.OP_NOOP
    req["profile"][kind == 7] = E.PROFILE_UNKNOWN
    req["op"][kind == 7] = E.OP_ALLOC
    req[n - 1] = (n - 1, 15, E.OP_ALLOC, 0, 0)
    return req


def churn_batches(rng, ref, sizes, n_profiles, frees=3, others=None):
    """Batches of the given sizes: ALLOCs of every profile and of an unknown one, up to 1/``frees`` of them replaced by FREEs of live
    allocations.  Returns [(requests, ``ref``'s results)]; ``others`` are placed the same batches too and must agree with ``ref``."""
    batches, live = [], []
    for n in sizes:
        req = W.alloc_requests((rng.next(n) % np.uint64(n_profiles + 1)).astype(np.uint8))
        req["profile"][req["profile"] == n_profiles] = E.PROFILE_UNKNOWN
        for _ in range(min(len(live), n // frees)):
            g, s, z = live.pop(int(rng.next1() % len(live)))
            req[int(rng.next1() % n)] = (g, 0, E.OP_FREE, s, z)
        res = ref.place(req)
        for other in others or ():
            assert np.array_equal(other.place(req), res), (n, len(batches))
            assert np.array_equal(other.occupancy(), ref.occupancy()), (n, len(batches))
        live.extend((int(r["gpu"]), int(r["start"]), int(r["size"])) for r in res[(req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)])
        batches.append((req, res))
    return batches


def default_sizes(rows2d, node_table):
    """Size an unplaced request of each name reports: the row of the first node in canonical order whose table knows the name."""
    out = []
    for p in range(rows2d.shape[1]):
        t = next((int(t) for t in node_table if rows2d["n_starts"][t, p]), None)
        out.append(0 if t is None else int(rows2d["size"][t, p]))
    return out


# ---- self-checks: every fixture reaches the edge it is for ---------------------------------------------------------------------------
@pytest.mark.parametrize("quirks", QUIRK_SETS)
def test_t16x8_has_128_candidates_and_profile_15(quirks):
    rows = t16x8()
    cand = candidates(rows, quirks)
    assert len(rows) == E.MAX_PROFILES and len(cand) == 128 and cand_slots(len(cand)) == 4
    assert all(int(r["n_starts"]) == E.MAX_STARTS for r in rows)
    assert len({tuple(r["starts"]) for r in rows}) == 16                      # every row has its own order
    assert (65535 << 15 | 15 << 11) == 0x7FFFF800                               # the last key of a full chunk: bits 11..30 all set
    # a real key can never be INF: order 7 needs 8 legal starts, i.e. size 1, i.e. a one-bit mask
    assert max(bin(m).count("1") for _, _, _, m in cand) == 1


@pytest.mark.parametrize("quirks", QUIRK_SETS)
def test_t16mix_candidate_counts_select_k1_and_k2(quirks):
    for variant, k in ((1, 1), (2, 2)):
        rows = t16mix(variant)
        cand = candidates(rows, quirks)
        assert len(rows) == 16 and cand_slots(len(cand)) == k, (variant, len(cand))
        assert not [c for c in cand if c[1] == 15]                              # row 15: no quirk set places it
        assert len([c for c in cand if c[1] == 0]) == 8                         # a size-1 row with order 7
    rows = t16mix(2)
    assert {int(r["size"]) for r in rows} == set(range(1, 9))
    assert any(list(r["starts"][:r["n_starts"]]) != sorted(r["starts"][:r["n_starts"]]) for r in rows)
    assert any(int(s) + int(r["size"]) > 8 for r in rows for s in r["starts"][:r["n_starts"]])
    if quirks == E.QUIRKS_FIXED:            # odd sizes only place with the pow2 quirk off
        assert {bin(m).count("1") for _, _, _, m in candidates(rows, quirks)} == set(range(1, 9))


def test_t8tab_sits_at_128_candidates_with_more_than_32_big_ones():
    rows = t8tab()
    assert rows.shape == (8, 16)
    cand = candidates(rows, E.QUIRKS_FIXED)
    assert len(cand) == 128
    assert len(candidates(plus_one_candidate(rows, E.QUIRKS_FIXED), E.QUIRKS_FIXED)) == 129
    assert len([c for c in cand if bin(c[3]).count("1") >= 4]) > 32             # more than the 32 the speculative prologue keeps
    assert {bin(m).count("1") for _, _, _, m in cand} >= {3, 5, 6, 7}            # odd sizes
    assert {t for t, _, _, _ in cand} == set(range(8))
    known = rows["n_starts"] > 0
    assert not known.all(axis=1).any()                                          # every table is sparse
    assert known[:, 15].tolist() == [False] * 7 + [True]                        # profile 15: table 7 only ...
    assert [c for c in cand if c[1] == 15]                                      # ... and placeable there
    node_table = t8tab_node_tables(W.SplitMix64(1), 200)
    assert node_table[0] != 7 and set(node_table.tolist()) == set(range(8))


def test_t16top_reaches_the_largest_min_frag_score():
    """With 128 candidates every row is size 1 with 8 starts (no other size has 8 legal starts), and a size-1 placement kills 16 pairs;
    a size-8 row leaves room for 120 more candidates.  So a score never reaches 128 (bit 31 of the best-fit key); 121 is the top."""
    rows = t16top()
    assert len(candidates(rows, E.QUIRKS_FIXED)) == 121
    assert min_frag_scores(rows, E.QUIRKS_FIXED).max() == 121
    assert min_frag_scores(t16x8(), E.QUIRKS_REF_EXACT).max() == 16


def test_edge65535_places_the_all_ones_key_next_to_exhausted_lanes():
    rows = t16x8()
    node_off, occ, req = edge65535(W.SplitMix64(65535))
    assert len(req) == EDGE_N and req["profile"][-1] == 15 and req["op"][-1] == E.OP_ALLOC
    ref = oracle.Fast(node_off, rows)
    ref.load(occ)
    res = ref.place(req)
    last = res[-1]
    assert last["status"] == E.ST_PLACED
    # a lane is exhausted when every request of its profile is placed on a GPU the chain has passed (at the GPU of the last request
    # those with a smaller index were decided first)
    alloc = req["op"] == E.OP_ALLOC
    exhausted = [p for p in range(15) if (alloc & (req["profile"] == p)).any()
                 and ((res["status"] == E.ST_PLACED) & (res["gpu"] <= last["gpu"]))[alloc & (req["profile"] == p)].all()]
    assert 3 in exhausted, exhausted
    assert (res["status"][alloc & (req["profile"] < 16)] == E.ST_PLACED).all()


def test_default_size_of_profile_15_comes_from_table_7():
    rows = t8tab()
    rng = W.SplitMix64(15)
    n_nodes = 40
    node_off = ragged_nodes(rng, n_nodes)
    node_table = t8tab_node_tables(rng, n_nodes)
    assert set(node_table.tolist()) == set(range(8))
    G = int(node_off[-1])
    want = default_sizes(rows, node_table)
    assert want[15] == int(rows["size"][7, 15]) and int(rows["n_starts"][node_table[0], 15]) == 0
    assert [p for p in range(16) if want[p] != int(rows["size"][node_table[0], p])]        # more than profile 15 is not node 0's
    full = np.full(G, 0xFF, dtype=np.uint8)
    req = W.alloc_requests(np.arange(16, dtype=np.uint8))
    for ref in (oracle.Fast(node_off, rows, 0, node_table=node_table), oracle.Faithful(node_off, rows, 0, node_table=node_table)):
        if isinstance(ref, oracle.Fast):
            ref.load(full)
        else:
            ref.load_occupancy_as_dangling(full)
        res = ref.place(req)
        assert (res["status"] == E.ST_NO_CAPACITY).all()
        assert res["size"].tolist() == want


# ---- the two C++ restatements agree at these shapes ----------------------------------------------------------------------------------
FIXTURES = {"t16x8": t16x8, "t16mix1": lambda: t16mix(1), "t16mix2": lambda: t16mix(2), "t16top": t16top, "t8tab": t8tab}


@pytest.mark.parametrize("quirks", QUIRK_SETS)
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_fast_vs_faithful_at_the_limits(name, quirks):
    """Ragged nodes, random occupancy, unknown profiles, frees of live allocations; per-node tables for T8tab."""
    rows = FIXTURES[name]()
    rng = W.SplitMix64(4000 + 10 * quirks + len(name))
    for trial in range(4):
        n_nodes = 1 + int(rng.next1() % 8)
        node_off = ragged_nodes(rng, n_nodes)
        G = int(node_off[-1])
        node_table = t8tab_node_tables(rng, n_nodes) if rows.ndim == 2 else None
        occ = ((rng.next(G) & rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
        fast = oracle.Fast(node_off, rows, quirks, node_table=node_table)
        fast.load(occ)
        faith = oracle.Faithful(node_off, rows, quirks, node_table=node_table)
        faith.load_occupancy_as_dangling(occ)
        churn_batches(rng, fast, [5 + int(rng.next1() % 60) for _ in range(4)], rows.shape[-1], others=[faith])


def test_fast_vs_faithful_on_the_edge_shape():
    """Edge65535's request mix (NOOPs, unknown profiles, profile 3 early only, profile 15 last) on a small inventory."""
    rows = t16x8()
    rng = W.SplitMix64(99)
    for n_nodes, n in ((3, 200), (9, 1500)):
        node_off = ragged_nodes(rng, n_nodes)
        G = int(node_off[-1])
        occ = (rng.next(G) & rng.next(G) & np.uint64(0xFF)).astype(np.uint8)
        req = edge_requests(rng, n)
        fast = oracle.Fast(node_off, rows)
        fast.load(occ)
        faith = oracle.Faithful(node_off, rows)
        faith.load_occupancy_as_dangling(occ)
        assert np.array_equal(fast.place(req), faith.place(req)), n
        assert np.array_equal(fast.occupancy(), faith.occupancy()), n
