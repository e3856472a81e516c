"""Times isl_place_gangs on an ISL_FLAG_GANG_FEW_NODES engine on the input of tools/gang_node_time.py: 8 192 nodes x 8 H100 GPUs,
pre-filled to about half of its slices by C3-mix pods of which every other one was released again, with 20 000 pods of the C3 mix cut
into gangs of 2, 4 and 8 consecutive requests, first-fit and best-fit.  Next to it: the same call on a GANG_ONE_NODE engine and on an
unflagged engine, and the brute force of tests/gang_few_fast.cpp (one core, the CPU baseline).

Outcome (--outcome-only runs on a machine without a GPU): placed members, aborted gangs and the mean number of nodes per committed gang
of the few-node, one-node and unflagged rules, from the brute forces.  Time: the median of --reps synchronous calls with CUDA events,
each printed only after the engine's records and final occupancy were found byte-identical to the brute force's.  One JSON line per
(policy, gang size); the card and its power limit are read in the same run.

    python tools/gang_few_time.py [--reps 5] [--outcome-only] [--out results/gang_few_time.json]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import oracle  # noqa: E402
from instaslice_b200 import engine as E, workloads as W  # noqa: E402
import gang_few_fast as GFF  # noqa: E402
import gang_node_fast as GNF  # noqa: E402
import gang_oracle as GO  # noqa: E402
from gang_node_time import card, prefilled, timed  # noqa: E402


def outcome(out, off, node_off):
    """placed members, aborted gangs, mean nodes per committed gang"""
    placed = out["status"] == E.ST_PLACED
    node = np.searchsorted(node_off, out["gpu"], side="right") - 1
    nodes, aborted = [], 0
    for a, b in zip(off[:-1], off[1:]):
        if (out["status"][a:b] == E.ST_GANG_ABORTED).any() or not placed[a:b].all():
            aborted += 1
        else:
            nodes.append(len(set(node[a:b].tolist())))
    return {"placed": int(placed.sum()), "aborted_gangs": aborted, "nodes_per_gang": round(float(np.mean(nodes)), 4) if nodes else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pods", type=int, default=20_000)
    ap.add_argument("--outcome-only", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rng = W.SplitMix64(42)
    node_off = W.node_offsets(8192, 8)
    rows = E.make_profiles(W.tables.H100_80GB)
    occ = prefilled(node_off, rows, rng)
    req = W.alloc_requests(W.mix_profiles(rng, args.pods))
    lines = []
    if not args.outcome_only:
        import torch
        info = card()
        stream = torch.cuda.Stream()
    for policy, pname in ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit")):
        engines = {}
        if not args.outcome_only:
            for flags in (E.FLAG_GANG_FEW_NODES, E.FLAG_GANG_ONE_NODE, 0):
                eng = E.Engine(max_gpus=int(node_off[-1]), max_batch=len(req), policy=policy, flags=flags)
                eng.set_stream(stream.cuda_stream)
                eng.load_profiles(rows)
                engines[flags] = eng
        for k in (2, 4, 8):
            off = np.r_[np.arange(0, len(req), k), len(req)].astype(np.uint32)
            t0 = time.process_time()
            few, occ_few = GFF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
            cpu_ms = (time.process_time() - t0) * 1e3
            one, occ_one = GNF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
            ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
            ref.load(occ)
            plain = GO.fast_place_gangs(ref, req, off, GO.default_sizes(rows))
            line = {"policy": pname, "gang_size": k, "n_gangs": len(off) - 1, "requests": len(req), "gpus": int(node_off[-1]),
                    "nodes": len(node_off) - 1, "busy_slices": int(np.unpackbits(occ).sum()),
                    "few_nodes": outcome(few, off, node_off), "one_node": outcome(one, off, node_off),
                    "unflagged": outcome(plain, off, node_off), "brute_force_cpu_ms": round(cpu_ms, 1)}
            if not args.outcome_only:
                for flags, key, want, occ_want in ((E.FLAG_GANG_FEW_NODES, "few_nodes", few, occ_few),
                                                   (E.FLAG_GANG_ONE_NODE, "one_node", one, occ_one), (0, "unflagged", plain, ref.occupancy())):
                    eng = engines[flags]
                    ev_ms, host_ms, got = timed(eng, stream, lambda: eng.place_gangs(req, off), node_off, occ, args.reps)
                    assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), occ_want), (pname, k, key)
                    line[key + "_ms_events"], line[key + "_ms_host"] = round(ev_ms, 3), round(host_ms, 3)
                line.update(identical_to_brute_force=True, **info)
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
