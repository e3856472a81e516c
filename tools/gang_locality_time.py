"""Times isl_place_gangs on an ISL_FLAG_GANG_LOCALITY engine on the inventory of tools/gang_node_time.py (8 192 nodes x 8 H100 GPUs,
pre-filled to about half of its slices by C3-mix pods of which every other one was released again), with 20 000 C3-mix pods cut into
gangs of 2, 4 and 8 whose localities are drawn per gang from a seed.  Per (policy, gang size) one JSON line with:

  flagged     one call on the flagged engine (k_ganglocal);
  four_engines  what a caller does without the flag: four engines, one flagged for each locality (none for 0), one call per run of
              consecutive gangs of one locality, and the whole occupancy handed from each engine to the next between runs
              (isl_read_occupancy, isl_write_occupancy); host clock around the whole sequence;
  homogeneous every gang at locality k, on the flagged engine and on k's own engine (k_bestfit's gang loop for 0, k_gangnode,
              k_gangnode<true>, k_gangspread);
  brute force composition (i) of tests/gang_locality_oracle.py on one CPU core.

Medians of --reps synchronous calls, the inventory reloaded before each.  Every line is printed only after the flagged call's records and
final occupancy were found byte-identical to the composition's, and the four-engine sequence's to the flagged call's.  The card and its
power limit are read in the same run.

    python tools/gang_locality_time.py [--reps 5] [--out results/gang_locality_time.json]
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
import gang_locality_oracle as GLO  # noqa: E402
from gang_node_time import card, prefilled, timed  # noqa: E402

NAMES = {E.GANG_ANY_NODES: "any", E.GANG_ONE_NODE: "one_node", E.GANG_FEW_NODES: "few_nodes", E.GANG_DISTINCT_NODES: "distinct"}


def four_engines(engines, req, off, locality, node_off, occ):
    """The call as runs of one locality over four engines with whole-occupancy hand-overs; returns (host ms, records, occupancy)."""
    for eng in engines.values():
        eng.load_inventory(node_off, occ)
    torch.cuda.synchronize()
    runs = []                                       # (locality, first gang, last gang + 1)
    for g, loc in enumerate(locality):
        if runs and runs[-1][0] == loc:
            runs[-1][2] = g + 1
        else:
            runs.append([int(loc), g, g + 1])
    out = np.empty(len(req), dtype=E.RESULT_DTYPE)
    t0 = time.perf_counter()
    cur, prev = None, None
    for loc, g0, g1 in runs:
        eng = engines[loc]
        if prev is not None and prev is not eng:
            eng.write_occupancy(0, cur)
        a, b = int(off[g0]), int(off[g1])
        out[a:b] = eng.place_gangs(req[a:b], off[g0:g1 + 1] - off[g0])
        cur, prev = eng.read_occupancy(), eng
    return (time.perf_counter() - t0) * 1e3, out, cur


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pods", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gang_locality_time.py measures on a GPU and found none")
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
        engines = {}
        for flags in (E.FLAG_GANG_LOCALITY, 0, E.FLAG_GANG_ONE_NODE, E.FLAG_GANG_FEW_NODES, E.FLAG_GANG_DISTINCT_NODES):
            eng = E.Engine(max_gpus=G, max_batch=args.pods, policy=policy, flags=flags)
            eng.set_stream(stream.cuda_stream)
            eng.load_profiles(rows)
            engines[flags] = eng
        flagged = engines[E.FLAG_GANG_LOCALITY]
        own = {loc: engines[GLO.FLAG_OF[loc]] for loc in GLO.LOCALITIES}
        for k in (2, 4, 8):
            req = W.alloc_requests(mix)
            off = np.r_[np.arange(0, len(req), k), len(req)].astype(np.uint32)
            locality = (rng.next(len(off) - 1) % np.uint64(4)).astype(np.int64)
            t0 = time.process_time()
            want, occ_want = GLO.fast_gangs_locality(node_off, rows, occ, GLO.with_locality(req, off, locality), off, E.QUIRKS_REF_EXACT,
                                                     policy)
            cpu_ms = (time.process_time() - t0) * 1e3
            ev, host, got = timed(flagged, stream, lambda: flagged.place_gangs(req, off, locality), node_off, occ, args.reps)
            assert np.array_equal(got, want) and np.array_equal(flagged.read_occupancy(), occ_want), (pname, k)
            four = []
            for _ in range(args.reps):
                ms, got4, occ4 = four_engines(own, req, off, locality, node_off, occ)
                assert np.array_equal(got4, want) and np.array_equal(occ4, occ_want), (pname, k, "four engines")
                four.append(ms)
            homogeneous = {}
            for loc in GLO.LOCALITIES:
                same = [loc] * (len(off) - 1)
                h_ev, _, h_got = timed(flagged, stream, lambda: flagged.place_gangs(req, off, same), node_off, occ, args.reps)
                o_ev, _, o_got = timed(own[loc], stream, lambda: own[loc].place_gangs(req, off), node_off, occ, args.reps)
                assert np.array_equal(h_got, o_got), (pname, k, loc)
                homogeneous[NAMES[loc]] = {"flagged_ms_events": round(h_ev, 3), "own_engine_ms_events": round(o_ev, 3)}
            line = {"policy": pname, "gang_size": k, "n_gangs": len(off) - 1, "requests": len(req), "gpus": G, "nodes": len(node_off) - 1,
                    "busy_slices": int(np.unpackbits(occ).sum()), "gangs_per_locality": np.bincount(locality, minlength=4).tolist(),
                    "runs": int(1 + (np.diff(locality) != 0).sum()), "placed": int((want["status"] == E.ST_PLACED).sum()),
                    "flagged_ms_events": round(ev, 3), "flagged_ms_host": round(host, 3),
                    "four_engines_ms_host": round(float(np.median(four)), 3), "homogeneous": homogeneous,
                    "brute_force_cpu_ms": round(cpu_ms, 1), "identical_to_brute_force": True, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
        for eng in engines.values():
            eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
