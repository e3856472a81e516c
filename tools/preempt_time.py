"""Times isl_preempt on the config-4 inventory: 65 536 GPUs (8 192 nodes x 8) pre-filled to 50 % by workloads.Churn, every live
allocation listed as a victim with a SplitMix64 rank 0-7, and 1, 64 and 1 024 preemptors of the C3 mix at rank 8.

For each size: the synchronous call's time from CUDA events and from the host clock (medians), the same call through the brute-force
restatement of tests/preempt_fast.cpp on one CPU core, and a check that records and evict rows are byte-identical (a line is printed
only after it passed).  The card and its power limit are read in the same run.

    python tools/preempt_time.py [--reps 7] [--out results/preempt_time.json]
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
import preempt_fast as PF  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, _, watts = q.stdout.strip().partition(",") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit_w": float(watts) if watts.strip() else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    churn = W.Churn(n_nodes=8192, gpus_per_node=8, n_ops=0, fill=0.5)
    ref = oracle.Fast(churn.node_off, churn.rows)
    ref.load(np.zeros(churn.G, dtype=np.uint8))
    churn.generate(ref.place)
    occ = ref.occupancy()
    live = churn._live
    vic = np.zeros(live, dtype=E.VICTIM_DTYPE)
    vic["gpu"], vic["start"], vic["size"] = churn._gpu[:live], churn._start[:live], churn._size[:live]
    vic["priority"] = (W.SplitMix64(7).next(live) % np.uint64(8)).astype(np.uint8)
    info = card()
    eng = E.Engine(max_gpus=churn.G, max_batch=1024)
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    eng.load_profiles(churn.rows)
    eng.load_inventory(churn.node_off, occ)
    rng = W.SplitMix64(11)
    lines = []
    for n in (1, 64, 1024):
        req = W.alloc_requests(W.mix_profiles(rng, n))
        prio = np.full(n, 8, dtype=np.uint8)
        eng.preempt(req, prio, vic)                     # warm-up: buffers sized, modules loaded
        ev, host = [], []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            out, evict = eng.preempt(req, prio, vic)
            e1.record(stream)
            t1 = time.perf_counter()
            e1.synchronize()
            ev.append(e0.elapsed_time(e1))
            host.append((t1 - t0) * 1e3)
        t0 = time.process_time()
        rc, want, want_ev = PF.preempt(churn.node_off, churn.rows, occ, req, prio, vic)
        cpu_ms = (time.process_time() - t0) * 1e3
        assert rc == E.OK and np.array_equal(out, want) and np.array_equal(evict, want_ev), n
        assert np.array_equal(eng.read_occupancy(), occ)
        line = {"preemptors": n, "gpus": churn.G, "victims": live, "placed": int((out["status"] == E.ST_PLACED).sum()),
                "evicting": int((evict != E.GPU_NONE).any(axis=1).sum()), "ms_events": round(float(np.median(ev)), 4),
                "ms_host": round(float(np.median(host)), 4), "cpu_one_core_ms": round(cpu_ms, 2), "identical_to_checker": True, **info}
        print(json.dumps(line), flush=True)
        lines.append(line)
    eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
