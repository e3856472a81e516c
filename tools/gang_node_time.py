"""Times isl_place_gangs on an ISL_FLAG_GANG_ONE_NODE engine on a config-4-sized inventory (8 192 nodes x 8 H100 GPUs, pre-filled to
about half of its slices by C3-mix pods of which every other one was released again), with 20 000 pods of the C3 mix cut into gangs of
2, 4 and 8 consecutive requests.  Next to it: the same call on an unflagged engine (gangs spread over nodes, k_bestfit) and the brute
force of tests/gang_node_fast.cpp (one core, the CPU baseline).

Every line is printed only after the engine's records and final occupancy were found byte-identical to the brute force's.  One JSON
line per (policy, gang size); the card and its power limit are read in the same run.

    python tools/gang_node_time.py [--reps 7] [--out results/gang_node_time.json]
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

import oracle  # noqa: E402
from instaslice_b200 import engine as E, workloads as W  # noqa: E402
import gang_node_fast as GNF  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, _, watts = q.stdout.strip().partition(",") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit_w": float(watts) if watts.strip() else None}


def timed(eng, stream, call, node_off, occ, reps):
    """(median ms from CUDA events, median ms from the host clock) of a synchronous engine call on a freshly loaded inventory."""
    ev, host = [], []
    for _ in range(reps):
        eng.load_inventory(node_off, occ)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        out = call()
        e1.record(stream)
        t1 = time.perf_counter()
        e1.synchronize()
        ev.append(e0.elapsed_time(e1))
        host.append((t1 - t0) * 1e3)
    return float(np.median(ev)), float(np.median(host)), out


def prefilled(node_off, rows, rng):
    """C3-mix pods placed first-fit on the empty inventory, then every other one released: a fragmented, about half-full cluster."""
    G = int(node_off[-1])
    ref = oracle.Fast(node_off, rows)
    ref.load(np.zeros(G, dtype=np.uint8))
    res = ref.place(W.alloc_requests(W.mix_profiles(rng, G * 7 // 2)))
    live = res[res["status"] == E.ST_PLACED][::2]
    frees = np.zeros(len(live), dtype=E.REQUEST_DTYPE)
    frees["handle"], frees["op"], frees["start"], frees["size"] = live["gpu"], E.OP_FREE, live["start"], live["size"]
    ref.place(frees)
    return ref.occupancy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--pods", type=int, default=20_000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rng = W.SplitMix64(42)
    node_off = W.node_offsets(8192, 8)
    rows = E.make_profiles(W.tables.H100_80GB)
    occ = prefilled(node_off, rows, rng)
    req = W.alloc_requests(W.mix_profiles(rng, args.pods))
    info = card()
    lines = []
    stream = torch.cuda.Stream()
    for policy, pname in ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit")):
        engines = {}
        for flags in (E.FLAG_GANG_ONE_NODE, 0):
            eng = E.Engine(max_gpus=int(node_off[-1]), max_batch=len(req), policy=policy, flags=flags)
            eng.set_stream(stream.cuda_stream)
            eng.load_profiles(rows)
            engines[flags] = eng
        for k in (2, 4, 8):
            off = np.r_[np.arange(0, len(req), k), len(req)].astype(np.uint32)
            t0 = time.process_time()
            want, occ_want = GNF.place_gangs(node_off, rows, occ, req, off, E.QUIRKS_REF_EXACT, policy)
            cpu_ms = (time.process_time() - t0) * 1e3
            eng = engines[E.FLAG_GANG_ONE_NODE]
            ev_ms, host_ms, got = timed(eng, stream, lambda: eng.place_gangs(req, off), node_off, occ, args.reps)
            assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), occ_want), (pname, k)
            plain = engines[0]
            plain_ev, plain_host, _ = timed(plain, stream, lambda: plain.place_gangs(req, off), node_off, occ, args.reps)
            line = {"policy": pname, "gang_size": k, "n_gangs": len(off) - 1, "requests": len(req), "gpus": int(node_off[-1]),
                    "nodes": len(node_off) - 1, "busy_slices": int(np.unpackbits(occ).sum()),
                    "placed": int((got["status"] == E.ST_PLACED).sum()), "aborted": int((got["status"] == E.ST_GANG_ABORTED).sum()),
                    "one_node_ms_events": round(ev_ms, 3), "one_node_ms_host": round(host_ms, 3),
                    "unflagged_ms_events": round(plain_ev, 3), "unflagged_ms_host": round(plain_host, 3),
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
