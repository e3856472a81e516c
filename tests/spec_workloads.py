"""Structured workloads for the speculative rounds of k_pipeline (DESIGN.md 4.5), shared by the CPU tests (test_spec_workloads.py: the
oracles and the protocol model) and the device tests (test_gpu_spec_workloads.py).

The random tests feed i.i.d. request mixes over i.i.d. occupancy — the case the round-0 prediction was fitted to.  These workloads are
built to defeat the prediction and to reach the rarely taken branches of the correction: batches ordered by size, runs of one profile
whose length straddles the key-window margin, skewed groups and empty groups, queues that run dry at a stage boundary, occupancy
gradients and alternations aligned to the stage size or off by one GPU, stretches where only 1-slice spans fit, tables without a big
group or with a size-3 profile, node tables alternating stage by stage, batches of several chunks, FREEs only in the last stages.

Everything is deterministic (SplitMix64 seeds).  FREEs name allocations that are live when their batch starts, derived through
``oracle.Fast``.  ``worlds(w)`` states every batch of a single-table workload as an input of ``tests/spec_rounds_model.cpp --world``.
"""
from __future__ import annotations

import functools
import os
import subprocess
from dataclasses import dataclass

import numpy as np

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H100_SMS = 132          # SMs of an H100 SXM: one speculative stage per SM
WIN_MARGIN = 32         # kWinMargin (isl_kernels.cuh): queue entries staged on either side of a key window
CHUNK = 65536           # requests per pipeline chunk (kChunk): the device speculates a batch chunk by chunk
BASELINE_SEEDS = range(1, 13)   # an adversarial workload costs more model rounds than every one of these shuffles / permutations
H100 = E.make_profiles(tables.H100_80GB)
P1G, P1G20, P2G, P3G, P4G, P7G = range(6)           # row indices of tables.H100_80GB
BIG = (P3G, P4G, P7G)
SMALL = (P1G, P1G20, P2G)


def stage_size(G: int, sms: int = H100_SMS) -> int:
    """GPUs per stage of a single engine's speculative plan: segment_geometry aims at one stage per SM and rounds the segment up to a
    multiple of 64 GPUs, at least 64."""
    return max(64, (-(-G // sms) + 63) // 64 * 64)


@dataclass
class Workload:
    name: str
    rows: np.ndarray                    # [P] profile rows, or [T][P] with node_table
    quirks: int
    policy: int
    node_off: np.ndarray
    occ: np.ndarray
    batches: list
    node_table: np.ndarray | None = None
    baseline: str | None = None         # what the model compares against: "shuffle" the requests, "permute" the occupancy bytes
                                        # (each with every seed of BASELINE_SEEDS)
    edge: str = ""                      # no baseline: why the workload is kept as an edge-shape case

    @property
    def G(self) -> int:
        return int(self.node_off[-1])

    @property
    def single_table(self) -> bool:
        return self.rows.ndim == 1

    def oracle(self) -> oracle.Fast:
        ref = oracle.Fast(self.node_off, self.rows, self.quirks, self.policy, self.node_table)
        ref.load(self.occ)
        return ref

    def expected(self):
        """([results per batch], final occupancy) of the request-major oracle."""
        ref = self.oracle()
        return [ref.place(b) for b in self.batches], ref.occupancy()


# ---- building blocks -------------------------------------------------------------------------------------------------------------------
def _occ(rng, G, fill=0x7F):
    return ((rng.next(G) & rng.next(G)) & np.uint64(fill)).astype(np.uint8)


def _uniform(rng, n, n_profiles):
    return (rng.next(n) % np.uint64(n_profiles)).astype(np.uint8)


def _placed(req, res):
    keep = (req["op"] == E.OP_ALLOC) & (res["status"] == E.ST_PLACED)
    return [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in res[keep]]


def _frees(spans):
    req = np.zeros(len(spans), dtype=E.REQUEST_DTYPE)
    for i, (g, s, z) in enumerate(spans):
        req[i] = (g, 0, E.OP_FREE, s, z)
    return req


def _scatter(rng, allocs, frees):
    """FREEs placed at random positions among the ALLOCs (the engine applies a batch's FREEs first wherever they stand)."""
    req = np.concatenate([allocs, frees])
    return req[np.argsort(rng.next(len(req)), kind="stable")]


def _h100(name, G, occ, batches, **kw):
    return Workload(name, H100, E.QUIRKS_REF_EXACT, E.POLICY_FIRST_FIT, W.node_offsets(G // 8, 8), occ, batches, **kw)


def _layout(name, G, occ, seed, n=None, policy=E.POLICY_FIRST_FIT):
    rng = W.SplitMix64(seed)
    n = n if n is not None else G + G // 2
    w = _h100(name, G, occ, [W.alloc_requests(W.mix_profiles(rng, n))], baseline="permute")
    w.policy = policy
    return w


# ---- order inside a batch ------------------------------------------------------------------------------------------------------------
def order_big_first(G=8192):
    """All >= 4-slice requests first, then all 1g / 2g, each profile's requests in one run: the big group's heads move alone through
    the front, the small group's alone through the back, one profile at a time — the opposite of what the proportional round-0
    prediction assumes."""
    rng = W.SplitMix64(101)
    prof = W.mix_profiles(rng, G + G // 2)
    prof = prof[np.lexsort((prof, ~np.isin(prof, BIG)))]
    return _h100("order_big_first", G, _occ(rng, G), [W.alloc_requests(prof)], baseline="shuffle")


def order_small_first(G=8192):
    """The reverse: all 1g / 2g first, then all >= 4-slice requests, each profile's requests in one run."""
    rng = W.SplitMix64(102)
    prof = W.mix_profiles(rng, G + G // 2)
    prof = prof[np.lexsort((prof, np.isin(prof, BIG)))]
    return _h100("order_small_first", G, _occ(rng, G), [W.alloc_requests(prof)], baseline="shuffle")


def late_burst(G=8192):
    """An i.i.d. mix whose last 10 % is one big profile (3g): a burst the mass prediction spreads over the whole batch."""
    rng = W.SplitMix64(103)
    n = G + G // 2
    prof = W.mix_profiles(rng, n)
    prof[n - n // 10:] = P3G
    return _h100("late_burst", G, _occ(rng, G), [W.alloc_requests(prof)], baseline="shuffle")


def window_runs(run, G=8192):
    """Runs of one profile of length ``run`` (kWinMargin - 1, kWinMargin, kWinMargin + 1, 2 kWinMargin + 2), cycling through the six
    profiles: corrected entries land at the edges of the staged key windows."""
    rng = W.SplitMix64(104 + run)
    n = G + G // 2
    prof = ((np.arange(n) // run) % 6).astype(np.uint8)
    return _h100(f"window_runs_{run}", G, _occ(rng, G), [W.alloc_requests(prof)], baseline="shuffle")


# ---- skew inside a group -----------------------------------------------------------------------------------------------------------------
def skew_1g_2g(G=8192):
    """Tens of thousands of 1g requests and eight 2g: the 2g share rounds to nothing and the remainder rule carries the group."""
    rng = W.SplitMix64(201)
    n = 5 * G
    prof = np.full(n, P1G, dtype=np.uint8)
    prof[(rng.next(8) % np.uint64(n)).astype(np.int64)] = P2G
    return _h100("skew_1g_2g", G, _occ(rng, G), [W.alloc_requests(prof)], baseline="shuffle")


def small_group_without_1g(G=8192):
    """The small group is 1g.20gb and 2g.20gb (both 2 slices), no single-slice member: its last member takes the remainder."""
    rng = W.SplitMix64(202)
    prof = np.array([P1G20, P2G, P3G, P4G, P7G], dtype=np.uint8)[(rng.next(2 * G) % np.uint64(5)).astype(np.int64)]
    return _h100("small_group_without_1g", G, _occ(rng, G), [W.alloc_requests(prof)], baseline="shuffle")


def one_group_empty(G=8192):
    """Batches of big profiles only, then small only, then big only: one contention group is empty in every batch."""
    rng = W.SplitMix64(203)
    ref = oracle.Fast(W.node_offsets(G // 8, 8), H100)
    occ = _occ(rng, G)
    ref.load(occ)
    live, batches = [], []
    for b, group in enumerate((BIG, SMALL, BIG)):
        allocs = W.alloc_requests(np.array(group, dtype=np.uint8)[(rng.next(G) % np.uint64(len(group))).astype(np.int64)])
        k = min(len(live), G // 4)
        pick = [live.pop(int(rng.next1() % len(live))) for _ in range(k)]
        req = _scatter(rng, allocs, _frees(pick))
        live.extend(_placed(req, ref.place(req)))
        batches.append(req)
    return _h100("one_group_empty", G, occ, batches, edge="one group has no requests: the prediction degenerates to the other group")


# ---- exhaustion at a boundary ----------------------------------------------------------------------------------------------------------
def dry_at_stage_boundary(G=8192):
    """The 4g requests come last, and their number is sized with the oracle so that the last one is placed in the last stage before a
    stage boundary halfway through the inventory: the 4g queue runs dry exactly there, and every stage behind it must see an exhausted
    head."""
    rng = W.SplitMix64(301)
    occ = _occ(rng, G)
    prof = W.mix_profiles(rng, G + G // 2, mix=[("1g.10gb", 30), ("2g.20gb", 20), ("3g.40gb", 15), ("4g.40gb", 35)])
    prof = prof[np.argsort(prof == P4G, kind="stable")]
    sub = stage_size(G)
    res = _h100("", G, occ, []).oracle().place(W.alloc_requests(prof))
    gpus = res["gpu"][(prof == P4G) & (res["status"] == E.ST_PLACED)]
    boundary = (int(gpus[len(gpus) // 2]) // sub + 1) * sub
    keep = int(np.count_nonzero(gpus < boundary))
    prof = np.delete(prof, np.flatnonzero(prof == P4G)[keep:])
    return _h100("dry_at_stage_boundary", G, occ, [W.alloc_requests(prof)], baseline="shuffle")


def exactly_full(G=8192):
    """A batch whose every request is placed and that leaves no usable slice free: i.i.d. mix requests that fit, then exactly as many
    1g as free usable slices remain (slice 7 is unusable under the reference's strict bound)."""
    rng = W.SplitMix64(302)
    occ = _occ(rng, G)
    w = _h100("exactly_full", G, occ, [])
    ref = w.oracle()
    mix = W.alloc_requests(W.mix_profiles(rng, G))
    mix = mix[ref.place(mix)["status"] == E.ST_PLACED]
    free = int(np.unpackbits(~ref.occupancy() & np.uint8(0x7F)).sum())
    w.batches = [W.alloc_requests(np.concatenate([mix["profile"], np.full(free, P1G, dtype=np.uint8)]))]
    w.baseline = "shuffle"
    return w


# ---- occupancy layouts -------------------------------------------------------------------------------------------------------------------
def _stage_mask(G, pattern, shift=0):
    """Per GPU: pattern(stage index) over stages of stage_size(G) GPUs, moved ``shift`` GPUs towards the end."""
    sub = stage_size(G)
    return np.roll(np.array([pattern(g // sub) for g in range(G)], dtype=bool), shift)


def front_full_back_empty(G=8192, policy=E.POLICY_FIRST_FIT):
    """Front half of the stages full, back half empty: the first busy stage is far from stage 0."""
    S = -(-G // stage_size(G))
    occ = np.where(_stage_mask(G, lambda s: s < S // 2), 0xFF, 0).astype(np.uint8)
    tag = "_rtl" if policy == E.POLICY_RIGHT_TO_LEFT else ""
    return _layout("front_full_back_empty" + tag, G, occ, 401, policy=policy)


def front_empty_back_full(G=8192, policy=E.POLICY_FIRST_FIT):
    S = -(-G // stage_size(G))
    occ = np.where(_stage_mask(G, lambda s: s >= S // 2), 0xFF, 0).astype(np.uint8)
    tag = "_rtl" if policy == E.POLICY_RIGHT_TO_LEFT else ""
    return _layout("front_empty_back_full" + tag, G, occ, 402, policy=policy)


def alternating_stages(shift=0, G=8192):
    """Full and empty stages alternating, aligned to the stage size (shift 0) or off by one GPU."""
    occ = np.where(_stage_mask(G, lambda s: s % 2 == 0, shift), 0xFF, 0).astype(np.uint8)
    return _layout(f"alternating_stages_shift{shift}", G, occ, 403 + shift)


def hungry_stretches(G=8192):
    """Stretches where only 1-slice spans fit (0x7E: slice 0 free; 0x6D: slices 1 and 4 free) between empty stretches, neither aligned
    to the stage size: 1g heads move through the hungry stretches while every other head waits for the next empty one."""
    g = np.arange(G)
    occ = np.where((g % 176) < 144, np.where(g % 2 == 0, 0x7E, 0x6D), 0).astype(np.uint8)
    return _layout("hungry_stretches", G, occ, 405, n=2 * G)


def nothing_placeable(G=8192):
    """Every usable slice is busy: every stage is idle in every round."""
    w = _layout("nothing_placeable", G, np.full(G, 0x7F, dtype=np.uint8), 406)
    w.baseline, w.edge = None, "every occupancy byte is the same: no permutation differs"
    return w


# ---- tables --------------------------------------------------------------------------------------------------------------------------------
def a30(quirks, G=8192):
    """The A30 table (4 slices, 4g the only big profile) under either quirk set."""
    rng = W.SplitMix64(501 + quirks)
    rows = E.make_profiles(tables.A30_24GB)
    occ = _occ(rng, G, 0x0F)
    req = W.alloc_requests(_uniform(rng, 2 * G, len(rows)))
    return Workload(f"a30_quirks{quirks}", rows, quirks, E.POLICY_FIRST_FIT, W.node_offsets(G // 8, 8), occ, [req], baseline="permute")


SIZE3_TABLE = [("1g", 1, [0, 1, 2, 3, 4, 5, 6], 0), ("3s", 3, [0, 4, 1], 1), ("2g", 2, [0, 2, 4, 6], 2), ("4g", 4, [0, 4], 3)]
SIZE1_TABLE = [("a", 1, [0, 1, 2, 3, 4, 5, 6], 0), ("b", 1, [7, 6, 5, 4, 3, 2, 1, 0], 1), ("c", 1, [3, 4, 5], 2)]


def size3_fixed(G=8192):
    """A size-3 profile (placeable only under QUIRKS_FIXED) — it falls in the small group, whose mass counts slices."""
    rng = W.SplitMix64(503)
    rows = E.make_profiles(SIZE3_TABLE)
    req = W.alloc_requests(_uniform(rng, 2 * G, len(rows)))
    return Workload("size3_fixed", rows, E.QUIRKS_FIXED, E.POLICY_FIRST_FIT, W.node_offsets(G // 8, 8), _occ(rng, G, 0xFF), [req],
                    baseline="permute")


def size1_only(G=8192):
    """Size-1 profiles only: the big group is empty."""
    rng = W.SplitMix64(504)
    rows = E.make_profiles(SIZE1_TABLE)
    prof = _uniform(rng, 6 * G, len(rows))
    prof = prof[np.argsort(prof, kind="stable")]            # by profile: the heads of one profile at a time move
    return Workload("size1_only", rows, E.QUIRKS_REF_EXACT, E.POLICY_FIRST_FIT, W.node_offsets(G // 8, 8), _occ(rng, G, 0xFF), [W.alloc_requests(prof)],
                    baseline="shuffle")


def hetero_stage_blocks(G=8192):
    """H100 and A30 nodes alternating in blocks of exactly one stage."""
    rng = W.SplitMix64(505)
    names, rows = E.make_profile_tables([tables.H100_80GB, tables.A30_24GB])
    nodes_per_stage = stage_size(G) // 8
    node_table = ((np.arange(G // 8) // nodes_per_stage) % 2).astype(np.uint8)
    req = W.alloc_requests(_uniform(rng, 2 * G, len(names)))
    return Workload("hetero_stage_blocks", rows, E.QUIRKS_REF_EXACT, E.POLICY_FIRST_FIT, W.node_offsets(G // 8, 8), _occ(rng, G), [req],
                    node_table=node_table, edge="two node tables: the protocol model has no node map")


# ---- shape ---------------------------------------------------------------------------------------------------------------------------------
def many_chunks(n, G=16384):
    """One batch of several 65 536-request chunks: the chunks are speculated in sequence, each over the occupancy the last one left.
    The model sees them the same way, one world per chunk (``worlds``)."""
    rng = W.SplitMix64(600 + n)
    w = _h100(f"chunks_{n}", G, _occ(rng, G), [W.alloc_requests(W.mix_profiles(rng, n))])
    w.edge = "saturating i.i.d. mix: exercises the chunk sequence, not a prediction"
    return w


def free_heavy_tail(G=8192):
    """A saturating first batch, then batches that free every live span in the last eight stages (and only there) and allocate a mix:
    stage 0's prediction sees a full inventory that is empty at its far end.  Every batch's ALLOCs come one profile at a time (the FREE
    pattern alone costs about as many rounds as the same occupancy bytes permuted)."""
    rng = W.SplitMix64(701)
    occ = _occ(rng, G)
    w = _h100("free_heavy_tail", G, occ, [])
    ref = w.oracle()
    tail = G - 8 * stage_size(G)
    first = W.alloc_requests(np.sort(W.mix_profiles(rng, 3 * G), kind="stable"))
    live = _placed(first, ref.place(first))
    batches = [first]
    for b in range(2):
        pick = [x for x in live if x[0] >= tail]
        live = [x for x in live if x[0] < tail]
        req = _scatter(rng, W.alloc_requests(np.sort(W.mix_profiles(rng, len(pick)), kind="stable")), _frees(pick))
        live.extend(_placed(req, ref.place(req)))
        batches.append(req)
    w.batches = batches
    w.baseline = "permute"
    return w


BUILDERS = {
    "order_big_first": order_big_first,
    "order_small_first": order_small_first,
    "late_burst": late_burst,
    "window_runs_31": lambda G=8192: window_runs(WIN_MARGIN - 1, G),
    "window_runs_32": lambda G=8192: window_runs(WIN_MARGIN, G),
    "window_runs_33": lambda G=8192: window_runs(WIN_MARGIN + 1, G),
    "window_runs_66": lambda G=8192: window_runs(2 * WIN_MARGIN + 2, G),
    "skew_1g_2g": skew_1g_2g,
    "small_group_without_1g": small_group_without_1g,
    "one_group_empty": one_group_empty,
    "dry_at_stage_boundary": dry_at_stage_boundary,
    "exactly_full": exactly_full,
    "front_full_back_empty": front_full_back_empty,
    "front_empty_back_full": front_empty_back_full,
    "alternating_stages_shift0": lambda G=8192: alternating_stages(0, G),
    "alternating_stages_shift1": lambda G=8192: alternating_stages(1, G),
    "hungry_stretches": hungry_stretches,
    "nothing_placeable": nothing_placeable,
    "a30_quirks3": lambda G=8192: a30(E.QUIRKS_REF_EXACT, G),
    "a30_quirks0": lambda G=8192: a30(E.QUIRKS_FIXED, G),
    "size3_fixed": size3_fixed,
    "size1_only": size1_only,
    "hetero_stage_blocks": hetero_stage_blocks,
    "chunks_65537": lambda G=16384: many_chunks(65537, G),
    "chunks_131077": lambda G=16384: many_chunks(131077, G),
    "free_heavy_tail": free_heavy_tail,
    "front_full_back_empty_rtl": lambda G=8192: front_full_back_empty(G, E.POLICY_RIGHT_TO_LEFT),
    "front_empty_back_full_rtl": lambda G=8192: front_empty_back_full(G, E.POLICY_RIGHT_TO_LEFT),
}
NAMES = list(BUILDERS)
# Workloads that do not cost the model more rounds than every seeded baseline (tests/test_spec_workloads.py measures it): kept for the
# shape they give the device, not as adversaries of the prediction
EDGE_SHAPES = {
    "late_burst": "the burst lands behind the contended front: within the rounds of the shuffled batches",
    "window_runs_31": "within the rounds of the shuffled batches; corrections land one entry inside the staged window margin",
    "window_runs_32": "within the rounds of the shuffled batches; corrections land on the staged window margin",
    "window_runs_33": "within the rounds of the shuffled batches; corrections land one entry beyond the staged window margin",
    "window_runs_66": "within the rounds of the shuffled batches; runs span two window margins",
    "small_group_without_1g": "within the unbounded rounds of the shuffled batches (the bounded simulations take many more, DESIGN 4.5)",
    "exactly_full": "1g requests fill the last free slices behind the mix: fewer rounds than the shuffled batches",
    "front_full_back_empty": "a full front makes every stage's entry there the true one: fewer rounds than permuted bytes",
    "front_empty_back_full": "the batch is served before the full back half: within the rounds of permuted bytes",
    "alternating_stages_shift1": "one GPU of every full stage spills into the next: fewer rounds than permuted bytes",
    "hungry_stretches": "stages + 1 rounds, the same as permuted bytes: every stage is certified one round after the one in front",
    "a30_quirks3": "saturating uniform mix: stages - 1 rounds, within the rounds of permuted bytes",
    "a30_quirks0": "saturating uniform mix: stages - 1 rounds, within the rounds of permuted bytes",
    "size3_fixed": "saturating uniform mix: within the rounds of permuted bytes",
    "front_full_back_empty_rtl": "reversed storage puts the empty half in front: fewer rounds than permuted bytes",
    "front_empty_back_full_rtl": "reversed storage puts the full half in front: fewer rounds than permuted bytes",
}
# the four workloads with the most model rounds among those whose batches fit one open-stream slot (65 536 requests);
# test_spec_workloads.py keeps this list honest
HARDEST = ["hungry_stretches", "size1_only", "a30_quirks3", "a30_quirks0"]
# run on 2 and 3 ranks of one GPU at G = 4096
RANK_SUBSET = ["order_big_first", "window_runs_33", "alternating_stages_shift1", "hungry_stretches", "free_heavy_tail"]


@functools.lru_cache(maxsize=None)
def build(name: str, G: int | None = None) -> Workload:
    w = BUILDERS[name]() if G is None else BUILDERS[name](G=G)
    assert w.name == name
    if name in EDGE_SHAPES:
        w.baseline, w.edge = None, EDGE_SHAPES[name]
    return w


# ---- the protocol model's input ------------------------------------------------------------------------------------------------------------
def masks(rows, quirks):
    """Per profile: (size, slot masks in the order the start search tries them) — candidate_mask of isl_kernels.cuh restated."""
    out = []
    for row in rows:
        size, ms = int(row["size"]), []
        for v in row["starts"][:int(row["n_starts"])]:
            v = int(v)
            if v >= 8 or size == 0 or size > 8:
                continue
            if size > 1:
                if quirks & E.QUIRK_POW2_ONLY and size not in (2, 4, 8):
                    continue
                if (v + size >= 8) if quirks & E.QUIRK_STRICT_BOUND else (v + size > 8):
                    continue
            ms.append((((1 << size) - 1) << v) & 0xFF)
        out.append((size, ms))
    return out


@dataclass
class World:
    seg: int
    profiles: list          # [(size, [mask])]
    occ: np.ndarray         # in storage order: right-to-left stores the GPUs reversed
    times: np.ndarray       # [n] request time -> profile (255: no ALLOC)

    def text(self) -> str:
        lines = [f"{len(self.occ)} {self.seg} {len(self.profiles)}"]
        lines += [" ".join(map(str, [size, len(ms)] + ms)) for size, ms in self.profiles]
        lines.append(" ".join(map(str, self.occ.tolist())))
        for p in range(len(self.profiles)):
            t = np.flatnonzero(self.times == p)
            lines.append(" ".join(map(str, [len(t)] + t.tolist())))
        return "\n".join(lines) + "\n"

    def shuffled(self, seed):
        """The same requests in a random order."""
        rng = W.SplitMix64(seed)
        return World(self.seg, self.profiles, self.occ, self.times[np.argsort(rng.next(len(self.times)), kind="stable")])

    def permuted(self, seed):
        """The same occupancy bytes at random GPUs."""
        rng = W.SplitMix64(seed)
        return World(self.seg, self.profiles, self.occ[np.argsort(rng.next(len(self.occ)), kind="stable")], self.times)


def worlds(w: Workload, seg: int | None = None) -> list:
    """One model world per chunk, as the device speculates them: a batch is cut into chunks of CHUNK requests; the first sees the
    occupancy after the batch's FREEs, every later one the occupancy its predecessor left.  A world holds that occupancy and the
    chunk's ALLOCs by profile."""
    assert w.single_table
    seg = seg or stage_size(w.G)
    ref = w.oracle()
    prof = masks(w.rows, w.quirks)
    out = []
    for req in w.batches:
        occ = ref.occupancy()
        for r in req[req["op"] == E.OP_FREE]:
            occ[r["handle"]] &= np.uint8(~(((1 << int(r["size"])) - 1) << int(r["start"])) & 0xFF)
        for c0 in range(0, len(req), CHUNK):
            part = req[c0:c0 + CHUNK]
            times = np.where((part["op"] == E.OP_ALLOC) & (part["profile"] < len(prof)), part["profile"], 255).astype(np.uint8)
            out.append(World(seg, prof, occ[::-1].copy() if w.policy == E.POLICY_RIGHT_TO_LEFT else occ.copy(), times))
            step = oracle.Fast(w.node_off, w.rows, w.quirks, w.policy)
            step.load(occ)
            step.place(part[part["op"] == E.OP_ALLOC])
            occ = step.occupancy()
        ref.place(req)
        assert np.array_equal(occ, ref.occupancy())
    return out


def build_model(path: str) -> str:
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", path, os.path.join(ROOT, "tests", "spec_rounds_model.cpp")], check=True)
    return path


def run_model(exe: str, world: World, tmp: str, bounded: bool):
    """(exit code, stdout, rounds or None) of spec_rounds_model --world."""
    path = os.path.join(tmp, "world.txt")
    with open(path, "w") as f:
        f.write(world.text())
    out = subprocess.run([exe, "--world", path] + (["--bounded"] if bounded else []), capture_output=True, text=True)
    words = out.stdout.split()
    rounds = int(words[1]) if out.returncode == 0 and words[:1] == ["rounds"] else None
    return out.returncode, out.stdout, rounds
