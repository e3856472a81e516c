"""Times isl_place_gangs on an ISL_FLAG_GANG_DISTINCT_NODES engine on a config-4-sized inventory (8 192 nodes x 8 H100 GPUs, pre-filled
to about half of its slices by C3-mix pods of which every other one was released again, as tools/gang_node_time.py does), with 20 000
pods cut into gangs of 2, 4 and 8.  Two kinds of gang: "mix" (consecutive C3-mix pods) and "replicas" (k copies of one C3-mix profile).
Next to it: the same call on an unflagged engine (k_bestfit, gangs packed as close as the policy puts them), on an ISL_FLAG_GANG_ONE_NODE
engine (k_gangnode), and the brute force of tests/gang_spread_fast.cpp (one core, the CPU baseline).

Every line is printed only after the engine's records and final occupancy were found byte-identical to the brute force's.  One JSON
line per (policy, kind, gang size); the card and its power limit are read in the same run.

    python tools/gang_spread_time.py [--reps 7] [--out results/gang_spread_time.json]
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
import gang_spread_fast as GSF  # noqa: E402
from gang_node_time import card, prefilled, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--pods", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gang_spread_time.py measures on a GPU and found none")
    rng = W.SplitMix64(42)
    node_off = W.node_offsets(8192, 8)
    rows = E.make_profiles(W.tables.H100_80GB)
    occ = prefilled(node_off, rows, rng)
    mix = W.mix_profiles(rng, args.pods)
    info = card()
    lines = []
    stream = torch.cuda.Stream()
    for policy, pname in ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit")):
        engines = {}
        for flags in (E.FLAG_GANG_DISTINCT_NODES, E.FLAG_GANG_ONE_NODE, 0):
            eng = E.Engine(max_gpus=int(node_off[-1]), max_batch=args.pods, policy=policy, flags=flags)
            eng.set_stream(stream.cuda_stream)
            eng.load_profiles(rows)
            engines[flags] = eng
        for kind in ("mix", "replicas"):
            for k in (2, 4, 8):
                req = W.alloc_requests(mix if kind == "mix" else np.repeat(mix[::k], k)[:args.pods])
                off = np.r_[np.arange(0, len(req), k), len(req)].astype(np.uint32)
                t0 = time.process_time()
                want, occ_want = GSF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
                cpu_ms = (time.process_time() - t0) * 1e3
                ms = {}
                for flags, label in ((E.FLAG_GANG_DISTINCT_NODES, "distinct"), (E.FLAG_GANG_ONE_NODE, "one_node"), (0, "unflagged")):
                    eng = engines[flags]
                    ev, host, got = timed(eng, stream, lambda: eng.place_gangs(req, off), node_off, occ, args.reps)
                    ms[label] = (ev, host)
                    if flags == E.FLAG_GANG_DISTINCT_NODES:
                        assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), occ_want), (pname, kind, k)
                        placed = int((got["status"] == E.ST_PLACED).sum())
                line = {"policy": pname, "kind": kind, "gang_size": k, "n_gangs": len(off) - 1, "requests": len(req),
                        "gpus": int(node_off[-1]), "nodes": len(node_off) - 1, "busy_slices": int(np.unpackbits(occ).sum()),
                        "placed": placed, "distinct_ms_events": round(ms["distinct"][0], 3), "distinct_ms_host": round(ms["distinct"][1], 3),
                        "one_node_ms_events": round(ms["one_node"][0], 3), "unflagged_ms_events": round(ms["unflagged"][0], 3),
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
