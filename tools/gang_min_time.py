"""Times isl_place_gangs on an ISL_FLAG_GANG_MIN_MEMBERS engine on the inventory of tools/gang_node_time.py (8 192 nodes x 8 H100 GPUs,
pre-filled to about half of its slices by C3-mix pods of which every other one was released again), with 20 000 C3-mix pods cut into
gangs of k = 4, 8 and 16 with minimum m = k / 2, under first-fit and best-fit, for every gang flag with MIN: none (any), one node, few
nodes, distinct nodes and a locality per gang drawn from a seed.  Per (policy, mode, k) one JSON line with:

  flagged      one call on the MIN engine (k_ganglocal<per_gang, min_members>);
  emulation    what a caller does without the flag, on the engine without MIN, host clock, run once: snapshot, place the rest of the
               call, and at the first gang that aborted at f >= m' restore, place the gangs before it and that gang cut to f in one call,
               then go on from the next gang (isl_snapshot_occupancy / isl_restore_occupancy); stopped after --emulation-s seconds, in
               which case the line holds the time so far as a lower bound;
  counts       trimmed and aborted gangs, pods placed;
  m0           m = 0 on the MIN engine against the same call on the engine without MIN: the price of routing through
               k_ganglocal<per_gang, min_members>;
  brute force  tests/gang_min_fast.cpp on one CPU core.

Medians of --reps synchronous calls, the inventory reloaded before each.  Every line is printed only after the flagged call's records and
final occupancy were found byte-identical to the brute force's, and the emulation's (when it finished) and the m = 0 calls' to theirs.
The card and its power limit are read in the same run.

    python tools/gang_min_time.py [--reps 5] [--out results/gang_min_time.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from instaslice_b200 import engine as E, workloads as W  # noqa: E402
import gang_min_fast as GMF  # noqa: E402
from gang_node_time import card, prefilled, timed  # noqa: E402

MODES = [("any", 0, E.GANG_ANY_NODES), ("one_node", E.FLAG_GANG_ONE_NODE, E.GANG_ONE_NODE),
         ("few_nodes", E.FLAG_GANG_FEW_NODES, E.GANG_FEW_NODES), ("distinct", E.FLAG_GANG_DISTINCT_NODES, E.GANG_DISTINCT_NODES),
         ("locality", E.FLAG_GANG_LOCALITY, None)]


def emulation(eng, req, off, locality, m, node_off, occ, budget_s):
    """The elastic call on an engine without MIN by snapshot, call and restore; returns (host ms, records or None when stopped, calls)."""
    eng.load_inventory(node_off, occ)
    torch.cuda.synchronize()
    per_gang = locality if eng.flags & E.FLAG_GANG_LOCALITY else None
    n_gangs = len(off) - 1
    out = np.empty(len(req), dtype=E.RESULT_DTYPE)
    t0 = time.perf_counter()
    g, calls = 0, 0
    while g < n_gangs:
        if time.perf_counter() - t0 > budget_s:
            return (time.perf_counter() - t0) * 1e3, None, calls
        a = int(off[g])
        sub_off = off[g:] - off[g]
        eng.snapshot_occupancy()
        res = eng.place_gangs(req[a:], sub_off, None if per_gang is None else per_gang[g:])
        calls += 1
        placed = (res["status"] == E.ST_PLACED)
        j = None
        for h in range(n_gangs - g):                   # the first gang that aborted with f >= m'
            s = res["status"][sub_off[h]:sub_off[h + 1]]
            f = int(np.flatnonzero(s != E.ST_GANG_ABORTED)[0]) if not placed[sub_off[h]:sub_off[h + 1]].all() else None
            if f is not None and f >= (len(s) if m == 0 or m >= len(s) else m):
                j = h
                break
        if j is None:
            out[a:] = res
            break
        eng.restore_occupancy()
        cut_end = int(sub_off[j]) + f
        cut_off = np.r_[sub_off[:j + 1], cut_end].astype(np.uint32)
        res2 = eng.place_gangs(req[a:a + cut_end], cut_off, None if per_gang is None else per_gang[g:g + j + 1])
        calls += 1
        out[a:a + cut_end] = res2
        out[a + cut_end:a + int(sub_off[j + 1])] = res[cut_end:int(sub_off[j + 1])]
        out["status"][a + cut_end + 1:a + int(sub_off[j + 1])] = E.ST_GANG_TRIMMED
        g += j + 1
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out, calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pods", type=int, default=20_000)
    ap.add_argument("--emulation-s", type=float, default=20.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gang_min_time.py measures on a GPU and found none")
    rng = W.SplitMix64(42)
    node_off = W.node_offsets(8192, 8)
    rows = E.make_profiles(W.tables.H100_80GB)
    occ = prefilled(node_off, rows, rng)
    mix = W.mix_profiles(rng, args.pods)
    info = card()
    lines = []
    stream = torch.cuda.Stream()
    G = int(node_off[-1])
    for policy, pname in ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit")):
        for mname, flags, loc in MODES:
            elastic = E.Engine(max_gpus=G, max_batch=args.pods, policy=policy, flags=E.FLAG_GANG_MIN_MEMBERS | flags)
            plain = E.Engine(max_gpus=G, max_batch=args.pods, policy=policy, flags=flags)
            for eng in (elastic, plain):
                eng.set_stream(stream.cuda_stream)
                eng.load_profiles(rows)
            for k in (4, 8, 16):
                req = W.alloc_requests(mix)
                off = np.r_[np.arange(0, len(req), k), len(req)].astype(np.uint32)
                n_gangs = len(off) - 1
                locality = (rng.next(n_gangs) % np.uint64(4)).astype(np.int64) if loc is None else np.full(n_gangs, loc, np.int64)
                per_gang = locality if flags & E.FLAG_GANG_LOCALITY else None
                minima = np.full(n_gangs, k // 2, dtype=np.int64)
                req_m = req.copy()
                req_m["size"] = k // 2
                t0 = time.process_time()
                want, occ_want, placed = GMF.place_gangs(node_off, rows, occ, req_m, off, locality, E.QUIRKS_REF_EXACT, policy)
                cpu_ms = (time.process_time() - t0) * 1e3
                ev, host, got = timed(elastic, stream, lambda: elastic.place_gangs(req, off, per_gang, minima), node_off, occ, args.reps)
                assert np.array_equal(got, want) and np.array_equal(elastic.read_occupancy(), occ_want), (pname, mname, k)
                emu_ms, emu, calls = emulation(plain, req, off, locality, k // 2, node_off, occ, args.emulation_s)
                if emu is not None:
                    assert np.array_equal(emu, want) and np.array_equal(plain.read_occupancy(), occ_want), (pname, mname, k, "emulation")
                z_ev, _, z_got = timed(elastic, stream, lambda: elastic.place_gangs(req, off, per_gang, np.zeros(n_gangs, np.int64)),
                                       node_off, occ, args.reps)
                p_ev, _, p_got = timed(plain, stream, lambda: plain.place_gangs(req, off, per_gang), node_off, occ, args.reps)
                assert np.array_equal(z_got, p_got), (pname, mname, k, "m = 0")
                per = np.add.reduceat(want["status"] == E.ST_PLACED, off[:-1].astype(np.int64))     # placed members per gang
                trimmed = int(((per > 0) & (per < np.diff(off))).sum())
                aborted = int((per == 0).sum())
                line = {"policy": pname, "mode": mname, "gang_size": k, "min_members": k // 2, "n_gangs": n_gangs, "requests": len(req),
                        "gpus": G, "nodes": len(node_off) - 1, "busy_slices": int(np.unpackbits(occ).sum()),
                        "trimmed_gangs": trimmed, "aborted_gangs": aborted, "placed": placed,
                        "flagged_ms_events": round(ev, 3), "flagged_ms_host": round(host, 3),
                        ("emulation_ms_host" if emu is not None else "emulation_ms_host_at_least"): round(emu_ms, 1),
                        "emulation_calls": calls, "m0_flagged_ms_events": round(z_ev, 3), "m0_without_min_ms_events": round(p_ev, 3),
                        "brute_force_cpu_ms": round(cpu_ms, 1), "identical_to_brute_force": True, **info}
                print(json.dumps(line), flush=True)
                lines.append(line)
            elastic.close()
            plain.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
