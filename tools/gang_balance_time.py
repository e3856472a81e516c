"""Times isl_place_gangs on an ISL_FLAG_GANG_LOCALITY | ISL_FLAG_GANG_BALANCED engine on the inventory of DESIGN.md 4.10 (8 192 nodes x
8 H100 GPUs, pre-filled to about half of its slices by C3-mix pods of which every other one was released again, as
tools/gang_spread_time.py does), with "replicas" gangs (k copies of one C3-mix profile) of 8, 16 and 32 at maxSkew 1 and 2.  Next to
them, on the same engine and input: byte 3 (distinct nodes) and byte 0 (any node), and the brute force of tests/gang_balance_fast.cpp
(one core, the CPU baseline).

Every line is printed only after the engine's records and final occupancy were found byte-identical to the brute force's, for every
byte it times.  Times are medians of --reps synchronous calls, by CUDA events and by the host clock; the card and its power limit are
read in the same run.  One JSON line per (policy, gang size, maxSkew).

    python tools/gang_balance_time.py [--reps 5] [--pods 4096] [--out results/gang_balance_time.json]
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
import gang_balance_fast as GBF  # noqa: E402
import gang_locality_oracle as GLO  # noqa: E402
from gang_node_time import card, prefilled, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pods", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gang_balance_time.py measures on a GPU and found none")
    rng = W.SplitMix64(42)
    node_off = W.node_offsets(8192, 8)
    rows = E.make_profiles(W.tables.H100_80GB)
    occ = prefilled(node_off, rows, rng)
    mix = W.mix_profiles(rng, args.pods)
    info = card()
    lines = []
    stream = torch.cuda.Stream()
    for policy, pname in ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit")):
        eng = E.Engine(max_gpus=int(node_off[-1]), max_batch=args.pods, policy=policy,
                       flags=E.FLAG_GANG_LOCALITY | E.FLAG_GANG_BALANCED)
        eng.set_stream(stream.cuda_stream)
        eng.load_profiles(rows)
        for k in (8, 16, 32):
            base = W.alloc_requests(np.repeat(mix[::k], k)[:args.pods])
            off = np.r_[np.arange(0, len(base), k), len(base)].astype(np.uint32)
            ms, cpu = {}, {}
            for byte in (0, 3, E.gang_balanced_nodes(1), E.gang_balanced_nodes(2)):
                req = GLO.with_locality(base, off, np.full(len(off) - 1, byte))
                t0 = time.process_time()
                want, occ_want, placed = GBF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
                cpu[byte] = (time.process_time() - t0) * 1e3
                ev, host, got = timed(eng, stream, lambda: eng.place_gangs(req, off), node_off, occ, args.reps)
                assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), occ_want), (pname, k, byte)
                ms[byte] = (ev, host, placed)
            for skew in (1, 2):
                b = E.gang_balanced_nodes(skew)
                line = {"policy": pname, "gang_size": k, "max_skew": skew, "n_gangs": len(off) - 1, "requests": len(base),
                        "gpus": int(node_off[-1]), "nodes": len(node_off) - 1, "busy_slices": int(np.unpackbits(occ).sum()),
                        "placed": ms[b][2], "balanced_ms_events": round(ms[b][0], 3), "balanced_ms_host": round(ms[b][1], 3),
                        "balanced_us_per_member": round(1e3 * ms[b][0] / len(base), 3),
                        "distinct_ms_events": round(ms[3][0], 3), "distinct_placed": ms[3][2],
                        "distinct_us_per_member": round(1e3 * ms[3][0] / len(base), 3),
                        "any_node_ms_events": round(ms[0][0], 3), "any_node_placed": ms[0][2],
                        "brute_force_cpu_ms": round(cpu[b], 1), "identical_to_brute_force": True, **info}
                print(json.dumps(line), flush=True)
                lines.append(line)
        eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
