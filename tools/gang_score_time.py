"""Times node-scored gangs (isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE engine, the node-scored k_ganglocal instantiations) on DESIGN.md
4.8's churn inventory: 65 536 GPUs in 7 669 nodes of 1 to 16 GPUs (SplitMix64 seed 5), every slice busy with probability 1/2, and
20 000 pods of the H100 mix cut into gangs of 2, 4 and 8 (SplitMix64 seed 13), for each locality and both policies.

Per (locality, policy): the flagged call's time from CUDA events and from the host clock (medians of --reps calls, the inventory
reloaded before each), the same pods through k_nodefit ungrouped (isl_place_batch on the same engine), the same gangs on a FIRST_FIT
engine with the same locality flag (k_bestfit's gang loop for any node, k_ganglocal otherwise), and the brute force of
tests/gang_score_fast.cpp on one CPU core.  A line is printed only after the flagged call's records, occupancy and stats.placed were
found byte-identical to the brute force.  The card and its power limit are read in the same run.

    python tools/gang_score_time.py [--reps 5] [--out results/gang_score_time.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from instaslice_b200 import engine as E, tables, workloads as W  # noqa: E402
import gang_score_fast as GSF  # noqa: E402

LOCALITIES = {"any_node": (E.GANG_ANY_NODES, 0), "one_node": (E.GANG_ONE_NODE, E.FLAG_GANG_ONE_NODE),
              "distinct_nodes": (E.GANG_DISTINCT_NODES, E.FLAG_GANG_DISTINCT_NODES)}
POLICIES = {"most_allocated": E.POLICY_MOST_ALLOCATED, "least_allocated": E.POLICY_LEAST_ALLOCATED}


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, _, watts = q.stdout.strip().partition(",") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit_w": float(watts) if watts.strip() else None}


def churn_inventory():
    """DESIGN.md 4.8's churn inventory (tools/node_score_time.py's, without its FREEs)."""
    rng = W.SplitMix64(5)
    sizes = (rng.next(20000) % np.uint64(16) + np.uint64(1)).astype(np.int64)
    sizes = sizes[:int(np.searchsorted(np.cumsum(sizes), 65536)) + 1]
    sizes[-1] -= int(sizes.sum()) - 65536
    node_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    bits = rng.next(65536 * 8).reshape(65536, 8) >> np.uint64(63)
    occ = (bits.astype(np.uint8) << np.arange(8, dtype=np.uint8)).sum(axis=1).astype(np.uint8)
    return node_off, occ, E.make_profiles(tables.H100_80GB)


def gang_call():
    """20 000 pods of the H100 mix in gangs of 2, 4 and 8 (the last gang takes what is left)."""
    rng = W.SplitMix64(13)
    req = W.alloc_requests(W.mix_profiles(rng, 20000))
    sizes = []
    for s in (2 << (rng.next(20000) % np.uint64(3))).astype(np.int64):
        if sum(sizes) >= len(req):
            break
        sizes.append(min(int(s), len(req) - sum(sizes)))
    return req, np.cumsum([0] + sizes).astype(np.uint32)


def timed(eng, stream, reps, node_off, occ, call):
    ev, host, out = [], [], None
    for rep in range(reps + 1):                         # the first call sizes the buffers and is not counted
        eng.load_inventory(node_off, occ)
        eng.reset_stats()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        out = call()
        e1.record(stream)
        t1 = time.perf_counter()
        e1.synchronize()
        if rep:
            ev.append(e0.elapsed_time(e1))
            host.append((t1 - t0) * 1e3)
    return out, round(float(np.median(ev)), 3), round(float(np.median(host)), 3)


def engine(policy, flags, rows, G, n, stream):
    eng = E.Engine(max_gpus=G, max_batch=n, policy=policy, flags=flags)
    eng.set_stream(stream.cuda_stream)
    eng.load_profiles(rows)
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = card()
    node_off, occ, rows = churn_inventory()
    req, off = gang_call()
    G, n = int(node_off[-1]), len(req)
    stream = torch.cuda.Stream()
    lines = []
    for lname, (loc, flag) in LOCALITIES.items():
        ff = engine(E.POLICY_FIRST_FIT, flag, rows, G, n, stream)
        _, ff_ev, _ = timed(ff, stream, args.reps, node_off, occ, lambda: ff.place_gangs(req, off))
        ff.close()
        for pname, policy in POLICIES.items():
            eng = engine(policy, E.FLAG_GANG_NODE_SCORE | flag, rows, G, n, stream)
            out, ms_ev, ms_host = timed(eng, stream, args.reps, node_off, occ, lambda: eng.place_gangs(req, off))
            occ_after, placed = eng.read_occupancy(), eng.stats()["placed"]
            t0 = time.process_time()
            want, occ_want, placed_want = GSF.place_gangs(node_off, rows, occ, req, off, policy, loc)
            cpu_ms = (time.process_time() - t0) * 1e3
            assert np.array_equal(out, want) and np.array_equal(occ_after, occ_want) and placed == placed_want, (lname, pname)
            _, nf_ev, _ = timed(eng, stream, args.reps, node_off, occ, lambda: eng.place_batch(req))
            n_gangs = len(off) - 1
            committed = sum(1 for a, b in zip(off[:-1], off[1:]) if (out["status"][a:b] == E.ST_PLACED).all())
            line = {"locality": lname, "policy": pname, "gangs": n_gangs, "pods": n, "gpus": G, "nodes": len(node_off) - 1,
                    "committed": committed, "placed": placed, "ms_events": ms_ev, "ms_host": ms_host,
                    "us_per_gang": round(ms_ev * 1e3 / n_gangs, 2), "k_nodefit_ungrouped_ms_events": nf_ev,
                    "first_fit_same_locality_ms_events": ff_ev, "cpu_one_core_ms": round(cpu_ms, 1), "identical_to_checker": True,
                    **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
            eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
