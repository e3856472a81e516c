"""One-node gangs (k_ganglocal<one_node>, ISL_FLAG_GANG_ONE_NODE) and distinct-node gangs (k_ganglocal<distinct_nodes>,
ISL_FLAG_GANG_DISTINCT_NODES) at the limits of the ABI — the layout restatement, the generators, their self-checks and the pins of the
checkers at these shapes (CPU only).  ``test_gpu_gang_topology_limits.py`` runs the same inputs through both kernels.

The fixtures are those of ``test_oracle_table_limits.py`` (T16x8, T16mix-1/2, T8tab with its node tables, T16top) and one more:
  T16straddle  15 size-4 rows of 5 starts and a size-2 row (index 15): profile 15's ISL_POLICY_MIN_FRAG score is 76 on an empty GPU,
               61 with slice 0 busy and 46 with slices 0 and 7 busy.  T16top's 121 is the largest score, but every GPU that admits its
               profile 15 is empty and scores exactly 121, so a member key that kept only the low 6 bits of the score would order
               those GPUs as before; here scores on both sides of 64 compete for one member.
Built here:
  gang_plan         gang_layout (islplace.cu) restated: the grid, every CTA's first node, the largest share, shared or global memory
  layout cases      a CTA that owns no node, as many nodes as the grid, a last CTA owning one one-GPU node, ceil(Gr / 512) limiting
                    the grid at 512 k and 512 k + 1 GPUs, a partition that cuts a node at both ends, one-node partitions on both sides
                    of the shared / global switch
  pass0_call        (one node) the first node in scan order that takes a gang has exactly the free slices the gang needs; a node
                    before it has as many free slices but cannot take the gang
  pass1_call        (one node) a gang's deepest failure is on a node that has fewer free slices than the gang needs
  dead15_call       (distinct nodes) profile 15 fails at rank >= 1 behind the exclusion (and is placed by the next gang), then at rank 0
                    (and stays dead for the call)
  min_frag_call     T16top / T16straddle under ISL_POLICY_MIN_FRAG: profile 15 scores 121, or scores on both sides of 64
  wrap_call         more than 510 gangs (the node-used tags wrap twice) on nodes of 64 GPUs, profile 15 placed after each wrap
"""
import time

import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import workloads as W

import gang_node_fast as GNF
import gang_node_oracle as GNO
import gang_oracle as GO
import gang_spread_fast as GSF
import gang_spread_oracle as GSO
from test_oracle_request_major_limits import (GANG_SHAPES, eight_gpu_nodes, fixture_migplacement, fixture_tables, gang_call, gang_offsets,
                                              names_of, node_tables_for, tables2, whole_bytes)
from test_oracle_table_limits import candidate_mask, candidates, min_frag_scores, t16mix, t16top, t16x8, t8tab, t8tab_node_tables

POLICIES = [E.POLICY_FIRST_FIT, E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_MIN_FRAG]
KERNELS = {"one_node": (E.FLAG_GANG_ONE_NODE, GNF.place_gangs), "distinct_nodes": (E.FLAG_GANG_DISTINCT_NODES, GSF.place_gangs)}
GN_MAX_CTAS = 160                   # kGnMaxCtas
GN_GPUS_PER_CTA = 512               # gang_layout: one CTA per 512 GPUs below one per SM
H100_SMS = 132
H100_OPTIN = 232448                 # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100 (227 KiB)
SM_COUNTS = (H100_SMS, 114, 78)


def t16straddle():
    return E.make_profiles([("w%d" % i, 4, [0, 1, 2, 3, 4], i) for i in range(15)] + [("pair", 2, [3], 15)])


FIXTURES = {"t16x8": t16x8, "t16mix1": lambda: t16mix(1), "t16mix2": lambda: t16mix(2), "t8tab": t8tab, "t16top": t16top,
            "t16straddle": t16straddle}
# (fixture, quirk set): T16mix under every quirk set, T8tab, T16top and T16straddle under FIXED quirks (their edges need them)
CASES = [("t16x8", E.QUIRKS_REF_EXACT)] + [(f, q) for f in ("t16mix1", "t16mix2") for q in (0, 1, 2, 3)] + \
        [(f, E.QUIRKS_FIXED) for f in ("t8tab", "t16top", "t16straddle")]


PIN_CASES = CASES + [("t16x8", q) for q in (0, 1, 2)]


def case_ids(cases):
    return ["%s-q%d" % c for c in cases]


# ---- gang_layout, restated ------------------------------------------------------------------------------------------------------------
class Plan:
    def __init__(self, grid, cta_node, shares, in_smem, nlo, nhi):
        self.grid, self.cta_node, self.shares, self.in_smem, self.nlo, self.nhi = grid, cta_node, shares, in_smem, nlo, nhi
        self.share = max(shares)


def gang_plan(node_off, lo, hi, sms, smem_optin, reverse=False):
    """gang_layout for the partition [lo, hi) (canonical) of ``node_off`` on a device of ``sms`` SMs whose gang kernels may have
    ``smem_optin`` bytes of dynamic shared memory (the device's opt-in minus their static shared memory).  ``reverse``: the
    right-to-left storage order.  The grid is min(SMs, kGnMaxCtas, ceil(Gr / 512), nodes the partition touches); CTA c owns the
    partition's nodes [cta_node[c], cta_node[c + 1]), cta_node[c] the first node that starts at or after lo + Gr c / grid; a share lives
    in shared memory when its two bytes per GPU, rounded up to 16 GPUs, fit in smem_optin (one 512-thread CTA per SM always fits
    there then)."""
    off = np.asarray(node_off, dtype=np.int64)
    G = int(off[-1])
    if reverse:
        off, lo, hi = G - off[::-1], G - hi, G - lo
    Gr = hi - lo
    nlo = int(np.searchsorted(off, lo, side="right")) - 1
    nhi = int(np.searchsorted(off, hi - 1, side="right"))
    grid = max(1, min(sms, GN_MAX_CTAS, -(-Gr // GN_GPUS_PER_CTA), nhi - nlo))
    cta = [0]
    for c in range(1, grid + 1):
        target = lo + Gr * c // grid
        cta.append(nhi - nlo if c == grid else int(np.searchsorted(off[nlo:nhi], target, side="left")))

    def local(j):
        return min(max(int(off[nlo + j]), lo), hi) - lo
    shares = [local(cta[c + 1]) - local(cta[c]) for c in range(grid)]
    return Plan(grid, cta, shares, (max(shares) + 15) // 16 * 16 * 2 <= smem_optin, nlo, nhi)


# ---- layout cases: (node_off, lo, hi) from the SM count -------------------------------------------------------------------------------
def offsets(sizes):
    return np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)


def cta_without_node(sms):
    """512 x SMs GPUs, the first node 1 536 of them: it spans the first three targets, so CTAs 1 and 2 own no node."""
    return offsets([1536] + [8] * ((512 * sms - 1536) // 8)), 0, 512 * sms


def nodes_equal_grid(sms):
    """SMs nodes of 512 GPUs: the grid is the node count and every CTA owns one node."""
    return offsets([512] * sms), 0, 512 * sms


def last_cta_one_gpu(sms):
    """512 (SMs - 1) + 1 GPUs: eight-GPU nodes, a node across the last target, and a one-GPU node that the last CTA owns alone."""
    G = 512 * (sms - 1) + 1
    target = G * (sms - 1) // sms
    b = target // 8 * 8 - 8
    return offsets([8] * (b // 8) + [G - 1 - b, 1]), 0, G


def grid_by_gpus(sms, extra):
    """512 k + extra GPUs in eight-GPU nodes, k = SMs / 2: ceil(Gr / 512) sets the grid (k, then k + 1)."""
    G = 512 * (sms // 2) + extra
    return eight_gpu_nodes(G), 0, G


def cut_both_ends(sms):
    """Nodes of 9..70 GPUs over about 512 x SMs + 3 000 GPUs, a partition that starts 7 GPUs into one node and ends 5 GPUs before the
    end of another."""
    rng = W.SplitMix64(sms)
    sizes = []
    while sum(sizes) < 512 * sms + 3000:
        sizes.append(9 + int(rng.next1() % 62))
    node_off = offsets(sizes)
    return node_off, int(node_off[3]) + 7, int(node_off[-4]) - 5


def one_node_partition(share):
    """A partition of ``share`` GPUs inside the middle one of three nodes, cutting it at both ends: one CTA holds all of it."""
    node_off = offsets([37, share + 16, 29])
    return node_off, 42, 42 + share


def smem_shares(optin):
    """Shares just below optin / 2 - 1 KiB (shared memory whatever the kernels' static shared memory up to 1 KiB) and just above
    optin / 2 (global memory)."""
    return optin // 2 - 1024 - 24, optin // 2 + 8


def layout_cases(sms, optin):
    """name -> (node_off, lo, hi, edge check on the plan at smem_optin = optin - static shared memory)."""
    below, above = smem_shares(optin)
    return {
        "cta_without_node": cta_without_node(sms) + (lambda p: p.grid == sms and 0 in p.shares,),
        "nodes_equal_grid": nodes_equal_grid(sms) + (lambda p: p.grid == sms == p.nhi - p.nlo and p.cta_node == list(range(sms + 1)),),
        "last_cta_one_gpu": last_cta_one_gpu(sms) + (lambda p: p.grid == sms and p.shares[-1] == 1 and p.cta_node[-1] - p.cta_node[-2] == 1,),
        "grid_512k": grid_by_gpus(sms, 0) + (lambda p: p.grid == sms // 2,),
        "grid_512k_plus_1": grid_by_gpus(sms, 1) + (lambda p: p.grid == sms // 2 + 1 and p.shares[-1] < 512,),
        "cut_both_ends": cut_both_ends(sms) + (lambda p: p.grid == sms,),
        "smem_below": one_node_partition(below) + (lambda p: p.grid == 1 and p.share == below and p.in_smem,),
        "smem_above": one_node_partition(above) + (lambda p: p.grid == 1 and p.share == above and not p.in_smem,),
    }


LAYOUT_CASES = list(layout_cases(H100_SMS, H100_OPTIN))


# ---- call generators ------------------------------------------------------------------------------------------------------------------
def first_mask(row, o, quirks):
    """Mask of the first legal start of ``row`` that is free on byte o, in row order; 0 for none."""
    for s in row["starts"][:row["n_starts"]]:
        m = int(candidate_mask(row["size"], s, quirks))
        if m and not o & m:
            return m
    return 0


def pack(rows2, t, members, quirks):
    """Masks the members take one after another on an empty byte of table t (first legal start each), or None when one finds none."""
    o, masks = 0, []
    for p in members:
        m = first_mask(rows2[t, p], o, quirks)
        if not m:
            return None
        o |= m
        masks.append(m)
    return masks


def scan_nodes(n_nodes, policy):
    return list(range(n_nodes - 1, -1, -1)) if policy == E.POLICY_RIGHT_TO_LEFT else list(range(n_nodes))


def packable_gang(rng, rows2, t, quirks, size, wide=1):
    """``size`` profiles of table t (fewer, down to 2, where the table has no such gang) that fit one empty byte together, the first
    ``wide`` of them two slices or more: (members, masks)."""
    known = [p for p in range(rows2.shape[1]) if rows2["n_starts"][t, p] and first_mask(rows2[t, p], 0, quirks)]
    for n in range(size, 1, -1):
        for _ in range(500):
            members = [known[int(rng.next1() % len(known))] for _ in range(n)]
            masks = pack(rows2, t, members, quirks)
            if masks and min(bin(m).count("1") for m in masks[:wide]) >= 2:
                return members, masks
    raise AssertionError("table %d has no such gang" % t)


def pass0_call(rng, policy, G=4096, n_gangs=6):
    """T8tab, FIXED quirks, eight-GPU nodes.  The first half of the nodes in scan order is full but for gang k's decoy node D_k and
    its perfect node X_k behind it (same table): X_k has one GPU whose free slices are exactly the masks the gang's members take, D_k
    as many free slices, one per GPU, which its first member (two slices or more) cannot use.  The second half has whole random bytes
    and every eighth node empty.  Returns (node_off, node_table, occ, req, gang_off, [(D_k, X_k)])."""
    rows = t8tab()
    quirks = E.QUIRKS_FIXED
    node_off = eight_gpu_nodes(G)
    n_nodes = len(node_off) - 1
    node_table = t8tab_node_tables(rng, n_nodes)
    scan = scan_nodes(n_nodes, policy)
    occ = whole_bytes(rng, G)
    for s, v in enumerate(scan):
        if s < n_nodes // 2:
            occ[node_off[v]:node_off[v + 1]] = 0xFF
        elif s % 8 == 0:
            occ[node_off[v]:node_off[v + 1]] = 0
    prof, off, pairs = [], [0], []
    for k in range(n_gangs):
        d, x = scan[10 + 30 * k], scan[20 + 30 * k]
        t = int(node_table[x])
        node_table[d] = t
        members, masks = packable_gang(rng, rows, t, quirks, 2 + k % 2)
        taken = int(np.bitwise_or.reduce(masks))
        g = int(node_off[x]) + int(rng.next1() % 8)
        occ[g] = 0xFF & ~taken
        need = bin(taken).count("1")
        for j in range(need):                                           # one free slice on each of `need` GPUs of D_k
            occ[int(node_off[d]) + j] = 0xFF & ~(1 << int(rng.next1() % 8))
        prof += members
        off.append(len(prof))
        pairs.append((d, x))
    req = W.alloc_requests(np.array(prof, dtype=np.uint8))
    return node_off, node_table, occ, req, np.asarray(off, dtype=np.uint32), pairs


def pass1_call(rng, policy, G=4096, n_gangs=3):
    """T8tab, FIXED quirks, eight-GPU nodes, every GPU one free slice.  Gang k = (a, b, c) fits nowhere: node Y_k has exactly a's and
    b's masks free on one GPU (depth 2, fewer free slices than the gang needs: pass 0 skips it), node Z_k has a's mask and spare single
    slices (depth 1, enough free slices: pass 0's winner); a and b take two slices or more.  Drawn again until no gang goes deeper on
    another gang's nodes.  Returns (node_off, node_table, occ, req, gang_off, [(Y_k, Z_k)])."""
    rows = t8tab()
    quirks = E.QUIRKS_FIXED
    node_off = eight_gpu_nodes(G)
    n_nodes = len(node_off) - 1
    scan = scan_nodes(n_nodes, policy)
    for _ in range(100):
        node_table = t8tab_node_tables(rng, n_nodes)
        occ = (0xFF & ~(np.uint64(1) << (rng.next(G) % np.uint64(8)))).astype(np.uint8)
        prof, off, pairs = [], [0], []
        for k in range(n_gangs):
            y, z = scan[300 + 40 * k], scan[100 + 40 * k]
            t = (2, 5, 6)[k]                                            # tables that have such gangs
            node_table[y] = node_table[z] = t
            members, masks = packable_gang(rng, rows, t, quirks, 3, wide=2)
            occ[node_off[y]:node_off[y + 1]] = 0xFF
            occ[int(node_off[y]) + 3] = 0xFF & ~(masks[0] | masks[1])
            occ[int(node_off[z])] = 0xFF & ~masks[0]
            prof += members
            off.append(len(prof))
            pairs.append((y, z))
        req = W.alloc_requests(np.array(prof, dtype=np.uint8))
        off = np.asarray(off, dtype=np.uint32)
        out, _ = GNF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table)
        if (out["status"].reshape(n_gangs, 3) == [E.ST_GANG_ABORTED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY]).all():
            return node_off, node_table, occ, req, off, pairs
    raise AssertionError("no pass-1 call found")


def dead15_call(rng, rows, quirks, G=4097, k=3):
    """Every GPU full but one GPU on each of k nodes (on table 7 for T8tab) with exactly profile 15's first mask free.  Gangs: 15 x
    (k + 1) (fails at rank k: every admitting node is used), 15 (placed), 15 x (k - 1) (placed), 15 (fails at rank 0: dead), 15 x 2 and
    15 (NO_CAPACITY at rank 0).  Returns (node_off, node_table, occ, req, gang_off, expected statuses per gang under the distinct-node
    rules)."""
    rows2 = tables2(rows)
    node_off = eight_gpu_nodes(G)
    n_nodes = len(node_off) - 1
    node_table = node_tables_for(rows, rng, n_nodes)
    nt = np.zeros(n_nodes, np.uint8) if node_table is None else node_table
    occ = np.full(G, 0xFF, dtype=np.uint8)
    picks = [int(v) for v in rng.next(k) % np.uint64(n_nodes)]
    assert len(set(picks)) == k
    t15 = 7 if rows2.shape[0] > 1 else 0
    for v in picks:
        nt[v] = t15
        occ[int(node_off[v]) + int(rng.next1() % int(node_off[v + 1] - node_off[v]))] = 0xFF & ~first_mask(rows2[t15, 15], 0, quirks)
    gangs = [[15] * (k + 1), [15], [15] * (k - 1), [15], [15] * 2, [15]]
    NC, AB, PL = E.ST_NO_CAPACITY, E.ST_GANG_ABORTED, E.ST_PLACED
    want = [[AB] * k + [NC], [PL], [PL] * (k - 1), [NC], [NC, AB], [NC]]
    req = W.alloc_requests(np.array([p for g in gangs for p in g], dtype=np.uint8))
    return node_off, node_table, occ, req, offsets([len(g) for g in gangs]), want


def min_frag_call(rng, name, G=4096, n=600):
    """T16top or T16straddle, eight-GPU nodes: every GPU empty, slice 0 busy, slices 0 and 7 busy, or full, so that profile 15 meets
    every score it has; gangs of 1..6 members, one in three profile 15."""
    rows = FIXTURES[name]()
    node_off = eight_gpu_nodes(G)
    kinds = np.array([0x00, 0x01, 0x81, 0xFF], dtype=np.uint8)
    occ = kinds[(rng.next(G) % np.uint64(4)).astype(np.int64)]
    prof = (rng.next(n) % np.uint64(15)).astype(np.uint8)
    prof[rng.next(n) % np.uint64(3) == 0] = 15
    req = W.alloc_requests(prof)
    return rows, node_off, occ, req, small_gangs(rng, n, 6)


def wrap_call(rng, n=1800):
    """T16x8, REF_EXACT quirks: 64 nodes of 64 GPUs, sparse whole bytes, gangs of 1..4 members (more than 510 gangs), profile 15 in
    each gang's last place one time in four."""
    rows = t16x8()
    node_off = offsets([64] * 64)
    occ = whole_bytes(rng, 4096)
    req = gang_call(rng, 4096, 16, n)
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % 4)))
        if rng.next1() % 4 == 0:
            req[off[-1] - 1] = (off[-1] - 1, 15, E.OP_ALLOC, 0, 0)
    return rows, node_off, occ, req, np.asarray(off, dtype=np.uint32)


def small_gangs(rng, n, most=4):
    """Offsets of gangs of 1..most requests: with T8tab's sparse tables and unknown profiles in the call, longer gangs rarely commit."""
    off = [0]
    while off[-1] < n:
        off.append(min(n, off[-1] + 1 + int(rng.next1() % most)))
    return np.asarray(off, dtype=np.uint32)


def lower_half_full(rng, G, n=200):
    """T8tab, eight-GPU nodes: the lower half of the inventory full but for what the call's FREEs release, the upper half dense whole
    bytes; gang_call's mix in gangs of 1..4."""
    rows = t8tab()
    node_off = eight_gpu_nodes(G)
    node_table = t8tab_node_tables(rng, len(node_off) - 1)
    occ = whole_bytes(rng, G, dense=True)
    occ[:G // 2] = 0xFF
    return rows, node_off, node_table, occ, gang_call(rng, G, 16, n), small_gangs(rng, n)


# ---- helpers of the self-checks -------------------------------------------------------------------------------------------------------
def node_of(node_off, g):
    return int(np.searchsorted(node_off, g, side="right")) - 1


def free_slices(occ, node_off, v):
    return int(sum(8 - bin(int(o)).count("1") for o in occ[node_off[v]:node_off[v + 1]]))


def need_of(rows2, t, members):
    return sum(int(rows2["size"][t, p]) for p in members)


def depth_on(rows, quirks, policy, occ, node_off, node_table, v, members):
    """How many leading members the one-node rules place on node v alone (len(members): all)."""
    rows2 = tables2(rows)
    one = np.array([0, node_off[v + 1] - node_off[v]], dtype=np.uint32)
    out, _ = GNF.place_gangs(one, rows2, occ[node_off[v]:node_off[v + 1]], W.alloc_requests(np.array(members, dtype=np.uint8)),
                             [0, len(members)], quirks, policy, np.array([node_table[v]], dtype=np.uint8))
    st = out["status"]
    return len(members) if (st == E.ST_PLACED).all() else int(np.flatnonzero(st != E.ST_GANG_ABORTED)[0])


def committed_nodes(out, req, off, node_off):
    """Per gang the nodes of its PLACED ALLOC members (empty for an aborted gang)."""
    res = []
    for a, b in zip(off[:-1], off[1:]):
        sel = (out["status"][a:b] == E.ST_PLACED) & (req["op"][a:b] == E.OP_ALLOC)
        res.append([node_of(node_off, int(g)) for g in out["gpu"][a:b][sel]])
    return res


# ---- the layout: gang_plan at its edges -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", SM_COUNTS)
def test_every_layout_case_reaches_its_edge(sms):
    for optin in (H100_OPTIN, 166912, 101376):
        for static in (0, 200, 1024):
            for name, (node_off, lo, hi, edge) in layout_cases(sms, optin).items():
                plan = gang_plan(node_off, lo, hi, sms, optin - static)
                assert edge(plan), (sms, optin, static, name, plan.grid, plan.shares[-3:])
                assert plan.cta_node[0] == 0 and plan.cta_node[-1] == plan.nhi - plan.nlo
                assert sum(plan.shares) == hi - lo and all(x >= 0 for x in plan.shares)


def test_cut_partition_cuts_a_node_at_both_ends():
    for sms in SM_COUNTS:
        node_off, lo, hi = cut_both_ends(sms)
        plan = gang_plan(node_off, lo, hi, sms, H100_OPTIN)
        assert node_off[plan.nlo] < lo < node_off[plan.nlo + 1] and node_off[plan.nhi - 1] < hi < node_off[plan.nhi]
        # right-to-left stores the inventory reversed: the same partition cuts the same two nodes, in the other order
        rev = gang_plan(node_off, lo, hi, sms, H100_OPTIN, reverse=True)
        assert rev.nhi - rev.nlo == plan.nhi - plan.nlo and rev.grid == plan.grid


def test_gang_plan_pins_the_shared_memory_switch():
    """Two bytes per GPU, the share rounded up to 16 GPUs: the largest share in shared memory is smem_optin / 32 * 16 GPUs."""
    for optin in (H100_OPTIN - 176, 232272, 1000):
        top = optin // 32 * 16
        for share, inside in ((top, True), (top + 1, False), (top - 15, True)):
            node_off, lo, hi = one_node_partition(share)
            assert gang_plan(node_off, lo, hi, H100_SMS, optin).in_smem == inside, (optin, share)


def test_gang_plan_at_2_20_gpus_and_the_top_partition():
    """2^20 GPUs of eight-GPU nodes: one CTA per SM, shares of about 7 944 GPUs in shared memory; the top partition [2^20 - 4 109, 2^20)
    cuts a node and is 9 CTAs wide, in either storage order."""
    G = 1 << 20
    node_off = eight_gpu_nodes(G)
    plan = gang_plan(node_off, 0, G, H100_SMS, H100_OPTIN)
    assert plan.grid == H100_SMS and plan.in_smem and 7900 < plan.share < 8000
    lo = G - 4096 - 13
    assert lo % 8 != 0
    for reverse in (False, True):
        top = gang_plan(node_off, lo, G, H100_SMS, H100_OPTIN, reverse)
        assert top.grid == 9 and sum(top.shares) == 4109


# ---- the call generators at their edges -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", POLICIES)
def test_pass0_call_puts_a_perfect_fit_first_behind_a_decoy(policy):
    rows2 = t8tab()
    rng = W.SplitMix64(600 + policy)
    for G in (4096, 4097):
        node_off, node_table, occ, req, off, pairs = pass0_call(rng, policy, G)
        out, _ = GNF.place_gangs(node_off, rows2, occ, req, off, E.QUIRKS_FIXED, policy, node_table)
        used = committed_nodes(out, req, off, node_off)
        for k, ((d, x), nodes) in enumerate(zip(pairs, used)):
            members = [int(p) for p in req["profile"][off[k]:off[k + 1]]]
            t = int(node_table[x])
            assert set(nodes) == {x}, (G, k, nodes, x)
            assert free_slices(occ, node_off, x) == need_of(rows2, t, members)         # a perfect fit ...
            assert free_slices(occ, node_off, d) == need_of(rows2, t, members)         # ... behind a decoy of as many free slices
            assert depth_on(rows2, E.QUIRKS_FIXED, policy, occ, node_off, node_table, d, members) < len(members)
            # without the perfect fit the gang commits on a later node: a filter that skipped X_k would be seen
            occ2 = occ.copy()
            occ2[node_off[x]:node_off[x + 1]] = 0xFF
            out2, _ = GNF.place_gangs(node_off, rows2, occ2, req[off[k]:off[k + 1]], [0, off[k + 1] - off[k]], E.QUIRKS_FIXED, policy,
                                      node_table)
            later = {node_of(node_off, int(g)) for g in out2["gpu"]}
            assert (out2["status"] == E.ST_PLACED).all() and len(later) == 1 and later != {x}
        assert {int(node_table[x]) for _, x in pairs} - {0, 1, 2}                         # tables beyond 0..2 (the & 3 mask reaches 4..7)
        assert max(int(b) - int(a) for a, b in zip(off[:-1], off[1:])) == 3


@pytest.mark.parametrize("policy", POLICIES)
def test_pass1_call_hides_the_deepest_failure_behind_the_filter(policy):
    rows2 = t8tab()
    rng = W.SplitMix64(700 + policy)
    node_off, node_table, occ, req, off, pairs = pass1_call(rng, policy)
    out, _ = GNF.place_gangs(node_off, rows2, occ, req, off, E.QUIRKS_FIXED, policy, node_table)
    for k, (y, z) in enumerate(pairs):
        members = [int(p) for p in req["profile"][off[k]:off[k + 1]]]
        st = out["status"][off[k]:off[k + 1]]
        assert st.tolist() == [E.ST_GANG_ABORTED, E.ST_GANG_ABORTED, E.ST_NO_CAPACITY], (k, st)     # depth 2: the third member
        t = int(node_table[y])
        assert free_slices(occ, node_off, y) < need_of(rows2, t, members)                          # pass 0 skips Y_k ...
        assert depth_on(rows2, E.QUIRKS_FIXED, policy, occ, node_off, node_table, y, members) == 2
        assert free_slices(occ, node_off, z) >= need_of(rows2, t, members)                         # ... and evaluates Z_k
        assert depth_on(rows2, E.QUIRKS_FIXED, policy, occ, node_off, node_table, z, members) == 1


@pytest.mark.parametrize("name,quirks", [("t16x8", E.QUIRKS_REF_EXACT), ("t8tab", E.QUIRKS_FIXED), ("t16top", E.QUIRKS_FIXED)])
@pytest.mark.parametrize("policy", POLICIES)
def test_dead15_call_fails_profile_15_behind_the_exclusion_then_at_rank_0(name, quirks, policy):
    rows = FIXTURES[name]()
    rng = W.SplitMix64(1500 + policy + len(name))
    node_off, node_table, occ, req, off, want = dead15_call(rng, rows, quirks)
    out, _ = GSF.place_gangs(node_off, rows, occ, req, off, quirks, policy, node_table)
    got = [out["status"][a:b].tolist() for a, b in zip(off[:-1], off[1:])]
    assert got == want
    assert int(req["profile"][off[1]]) == 15 and len(want[0]) >= 2                 # placed after a failure at rank >= 1


@pytest.mark.parametrize("name", ["t16top", "t16straddle"])
def test_min_frag_call_reaches_scores_above_63(name):
    rng = W.SplitMix64(121)
    rows, node_off, occ, req, off = min_frag_call(rng, name)
    score = min_frag_scores(rows, E.QUIRKS_FIXED)[15]
    fits = np.array([bool(first_mask(rows[15], int(o), E.QUIRKS_FIXED)) for o in range(256)])
    seen = sorted(set(int(score[o]) for o in np.unique(occ) if fits[o]))
    if name == "t16top":
        assert len(candidates(rows, E.QUIRKS_FIXED)) == 121 and seen == [121]
    else:
        assert len(candidates(rows, E.QUIRKS_FIXED)) == 76 and {46, 61, 76} <= set(seen)
        # a profile-15 member's choice by (score, position) differs from one by (score & 63, position): over the inventory (distinct
        # nodes), and inside most nodes (one node)
        def differ(g):
            return np.argmin(score[occ[g]] * (1 << 24) + g) != np.argmin((score[occ[g]] & 63) * (1 << 24) + g)
        g = np.flatnonzero(fits[occ])
        assert differ(g)
        inside = [differ(h) for v in range(len(node_off) - 1) if len(h := g[(g >= node_off[v]) & (g < node_off[v + 1])])]
        assert np.mean(inside) > 0.5
    for place in (GNF.place_gangs, GSF.place_gangs):
        out, _ = place(node_off, rows, occ, req, off, E.QUIRKS_FIXED, E.POLICY_MIN_FRAG)
        won = out[(req["profile"] == 15) & (out["status"] == E.ST_PLACED)]
        assert len(won) and set(int(score[occ[int(x)]]) for x in won["gpu"]) >= {min(seen)}


def test_wrap_call_places_profile_15_after_every_wrap():
    rng = W.SplitMix64(255)
    rows, node_off, occ, req, off = wrap_call(rng)
    assert len(off) - 1 > 2 * 255
    out, _ = GSF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, E.POLICY_FIRST_FIT)
    gang = np.searchsorted(off, np.arange(len(req)), side="right") - 1
    p15 = (req["op"] == E.OP_ALLOC) & (req["profile"] == 15) & (out["status"] == E.ST_PLACED)
    assert (gang[p15] >= 255).any() and (gang[p15] >= 510).any()
    used = committed_nodes(out, req, off, node_off)
    # a gang after the wrap reuses a node of the gang 255 before it, which had the same tag
    assert [i for i in range(255, len(used)) if set(used[i]) & set(used[i - 255])]


def test_lower_half_full_leaves_room_only_through_frees_below_2_19():
    rng = W.SplitMix64(19)
    G = 1 << 14                                         # the generator of the 2^20-GPU device test on a smaller inventory
    rows, node_off, node_table, occ, req, off = lower_half_full(rng, G, 400)
    for place in (GNF.place_gangs, GSF.place_gangs):
        out, _ = place(node_off, rows, occ, req, off, E.QUIRKS_FIXED, E.POLICY_FIRST_FIT, node_table)
        placed = out[(out["status"] == E.ST_PLACED) & (req["op"] == E.OP_ALLOC)]
        assert (placed["gpu"] >= G // 2).any() and (out["status"] == E.ST_GANG_ABORTED).any()


MEMO_CASES = [("t8tab", E.QUIRKS_FIXED), ("t16top", E.QUIRKS_FIXED), ("t16straddle", E.QUIRKS_FIXED), ("t16mix2", 1)]


# ---- the checkers against the restatements at the limits ------------------------------------------------------------------------------
def cluster(rng, rows, n_nodes):
    node_off = np.concatenate([[0], np.cumsum(1 + (rng.next(n_nodes) % np.uint64(3)).astype(np.int64))]).astype(np.uint32)
    node_table = node_tables_for(rows, rng, n_nodes)
    return node_off, node_table, whole_bytes(rng, int(node_off[-1]))


def crs_of(node_off, node_table, occ, rows):
    """One Instaslice dict per node whose Migplacement is the fixture's own (fixture_migplacement)."""
    nt = np.zeros(len(node_off) - 1, np.uint8) if node_table is None else node_table
    crs = GO.cluster_crs(node_off, nt, occ, fixture_tables(rows))
    migs = fixture_migplacement(rows)
    for n, cr in enumerate(crs):
        cr["spec"]["migplacement"] = migs[int(nt[n])]
    return crs


@pytest.mark.parametrize("name,quirks", PIN_CASES, ids=case_ids(PIN_CASES))
def test_brute_forces_agree_with_the_dict_restatements_first_fit(name, quirks):
    """First-fit: reconcile_gated_pod member by member on one node's resource (one-node) or on the cluster without the gang's nodes
    (distinct nodes), against the brute forces, verdict by verdict and occupancy after."""
    rows = FIXTURES[name]()
    names = names_of(rows)
    rng = W.SplitMix64(2000 + 10 * quirks + len(name))
    verdicts = {"one_node": set(), "distinct_nodes": set()}
    for trial in range(3):
        node_off, node_table, occ = cluster(rng, rows, 2 + int(rng.next1() % 7))
        gangs = [[int(rng.next1() % (len(names) + 1)) for _ in range(1 + int(rng.next1() % 4))] for _ in range(10)]
        req = W.alloc_requests(np.array([p if p < len(names) else E.PROFILE_UNKNOWN for g in gangs for p in g], dtype=np.uint8))
        off = offsets([len(g) for g in gangs])
        pods = [[({"uid": "u%d-%d" % (i, k), "name": "p", "namespace": "default"}, names[p] if p < len(names) else "unknown")
                 for k, p in enumerate(g)] for i, g in enumerate(gangs)]
        for kind, ref in (("one_node", GNO.ref_py_gangs_one_node), ("distinct_nodes", GSO.ref_py_gangs_distinct_nodes)):
            crs = crs_of(node_off, node_table, occ, rows)
            want = ref(crs, pods, quirks)
            got, after = KERNELS[kind][1](node_off, rows, occ, req, off, quirks, E.POLICY_FIRST_FIT, node_table)
            for gi, (verdict, detail) in enumerate(want):
                recs = got[off[gi]:off[gi + 1]]
                verdicts[kind].add(verdict)
                if verdict == "placed":
                    assert (recs["status"] == E.ST_PLACED).all(), (kind, trial, gi)
                    assert [(int(r["gpu"]), int(r["start"]), int(r["size"])) for r in recs] == \
                           [(int(a["gpuUUID"][4:]), a["start"], a["size"]) for a in detail], (kind, trial, gi)
                else:
                    assert int(np.flatnonzero(recs["status"] != E.ST_GANG_ABORTED)[0]) == detail, (kind, trial, gi)
                    assert (np.delete(recs["status"], detail) == E.ST_GANG_ABORTED).all(), (kind, trial, gi)
            assert np.array_equal(after, GO.cr_occupancy(crs)), (kind, trial)
    assert all(v == {"placed", "aborted"} for v in verdicts.values()), verdicts


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("name,quirks", PIN_CASES, ids=case_ids(PIN_CASES))
def test_brute_forces_agree_with_the_range_restatements(name, quirks, policy):
    """Every policy: the brute forces against the per-node RangeFast compositions of gang_node_oracle / gang_spread_oracle, on ragged
    clusters, whole bytes, every gang shape with FREEs, NOOPs and unknown profiles, whole inventories and cut partitions."""
    rows = FIXTURES[name]()
    rng = W.SplitMix64(3000 + 10 * quirks + 100 * policy + len(name))
    for trial, kind in enumerate(GANG_SHAPES):
        node_off, node_table, occ = cluster(rng, rows, 3 + int(rng.next1() % 10))
        G = int(node_off[-1])
        lo, hi = (0, G) if trial % 2 == 0 else (1 + int(rng.next1() % (G // 3)), G - 1 - int(rng.next1() % (G // 3)))
        n = 130 if kind == "straddle" else 60         # the straddling gang has up to 124 requests
        req = gang_call(rng, G, rows.shape[-1], n)
        off = gang_offsets(rng, kind, n)
        for brute, ranged in ((GNF.place_gangs, GNO.fast_gangs_one_node), (GSF.place_gangs, GSO.fast_gangs_distinct_nodes)):
            a, occ_a = brute(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
            b, occ_b = ranged(node_off, rows, occ, req, off, quirks, policy, node_table, lo, hi)
            bad = np.flatnonzero(a != b)
            assert len(bad) == 0, (brute.__module__, trial, bad[:4], a[bad[:4]], b[bad[:4]])
            assert np.array_equal(occ_a, occ_b), (brute.__module__, trial)


@pytest.mark.parametrize("name,quirks", MEMO_CASES, ids=case_ids(MEMO_CASES))
def test_memoised_min_frag_scores_agree_with_the_plain_walk(name, quirks):
    rows = FIXTURES[name]()
    rng = W.SplitMix64(4000 + len(name))
    placed = 0
    for G, shape in ((64, "ones"), (777, "mixed")):
        node_off = eight_gpu_nodes(G)
        node_table = node_tables_for(rows, rng, len(node_off) - 1)
        occ = whole_bytes(rng, G)
        req = gang_call(rng, G, rows.shape[-1], 300)
        off = gang_offsets(rng, shape, 300)
        for place in (GNF.place_gangs, GSF.place_gangs):
            a = place(node_off, rows, occ, req, off, quirks, E.POLICY_MIN_FRAG, node_table, 3, G - 2, memo=True)
            b = place(node_off, rows, occ, req, off, quirks, E.POLICY_MIN_FRAG, node_table, 3, G - 2, memo=False)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (place.__module__, G)
            placed += int((a[0]["status"] == E.ST_PLACED).sum())
    assert placed


def test_memoised_min_frag_is_affordable_at_2_20_gpus():
    """A distinct-node MIN_FRAG call over 2^20 GPUs on T16x8 (128 candidates): every member scores every GPU that admits it.  The
    plain walk counts up to 128 (profile, start) pairs per GPU and member; the memo walks each (table, profile, byte) once, which makes
    the call several times faster."""
    G = 1 << 20
    rng = W.SplitMix64(G)
    occ = whole_bytes(rng, G, dense=True)
    req = gang_call(rng, G, 16, 24)
    t0 = time.perf_counter()
    out, _ = GSF.place_gangs(eight_gpu_nodes(G), t16x8(), occ, req, small_gangs(rng, 24), E.QUIRKS_REF_EXACT, E.POLICY_MIN_FRAG)
    assert time.perf_counter() - t0 < 30
    assert (out["status"] == E.ST_PLACED).any()
