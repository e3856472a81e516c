"""Times isl_place_gangs on the C3 input (100 000 mixed-profile pods on 4 096 empty GPUs, seed 42) cut into gangs of 1, 4 and 16
consecutive requests, under ISL_POLICY_FIRST_FIT and ISL_POLICY_BEST_FIT, next to the same input through isl_place_batch and next to
the CPU restatement (tests/gang_oracle.py over ref_fast, one core, its Python loop over the gangs included).

Every line is printed only after the engine's records and final occupancy were found byte-identical to the restatement's.  One JSON
line per (policy, gang size); the card and its power limit are read in the same run.

    python tools/gang_time.py [--reps 7] [--out results/gang_time.json]
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
import gang_oracle as GO  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    node_off, occ, rows, req = W.config3()
    sizes = GO.default_sizes(rows)
    info = card()
    lines = []
    stream = torch.cuda.Stream()
    for policy, pname in ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit")):
        eng = E.Engine(max_gpus=int(node_off[-1]), max_batch=len(req), policy=policy)
        eng.set_stream(stream.cuda_stream)
        eng.load_profiles(rows)
        ref = oracle.Fast(node_off, rows, E.QUIRKS_REF_EXACT, policy)
        ref.load(occ)
        want_batch = ref.place(req)
        occ_batch = ref.occupancy()
        batch_ev, batch_host, got = timed(eng, stream, lambda: eng.place_batch(req), node_off, occ, args.reps)
        assert np.array_equal(got, want_batch) and np.array_equal(eng.read_occupancy(), occ_batch), (pname, "isl_place_batch")
        for k in (1, 4, 16):
            off = np.r_[np.arange(0, len(req), k), len(req)].astype(np.uint32)
            ref.load(occ)
            t0 = time.process_time()
            want = GO.fast_place_gangs(ref, req, off, sizes)
            cpu_ms = (time.process_time() - t0) * 1e3
            ev_ms, host_ms, got = timed(eng, stream, lambda: eng.place_gangs(req, off), node_off, occ, args.reps)
            assert np.array_equal(got, want) and np.array_equal(eng.read_occupancy(), ref.occupancy()), (pname, k)
            line = {"policy": pname, "gang_size": k, "n_gangs": len(off) - 1, "requests": len(req), "gpus": int(node_off[-1]),
                    "placed": int((got["status"] == E.ST_PLACED).sum()), "aborted": int((got["status"] == E.ST_GANG_ABORTED).sum()),
                    "gangs_ms_events": round(ev_ms, 3), "gangs_ms_host": round(host_ms, 3),
                    "batch_ms_events": round(batch_ev, 3), "batch_ms_host": round(batch_host, 3),
                    "oracle_cpu_ms": round(cpu_ms, 1), "identical_to_oracle": True, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
        eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
