"""Times node scoring (ISL_POLICY_MOST_ALLOCATED / _LEAST_ALLOCATED, k_nodefit) against ISL_POLICY_BEST_FIT (k_bestfit) on the same
inputs, and the brute-force restatement of tests/node_score_fast.cpp on one CPU core.

Inputs:
  c3     BASELINE config 3: 100 000 pods of the H100 mix (seed 42) on 512 empty 8-GPU nodes
  churn  a config-4-sized inventory: 65 536 GPUs in nodes of 1 to 16 GPUs (SplitMix64 seed 5), every slice busy with probability
         1/2, and one batch of 20 000 pods of the H100 mix with 2 000 single-slice FREEs in front of them

For each input and policy: the synchronous isl_place_batch's time from CUDA events and from the host clock (medians of --reps calls,
the inventory reloaded before each), the checker's time for the same batch, and a check that every record and the final occupancy are
byte-identical to the checker (node scoring) or to the CPU oracle (best-fit); a line is printed only after it passed.  The card and
its power limit are read in the same run.

    python tools/node_score_time.py [--reps 7] [--out results/node_score_time.json]
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
from instaslice_b200 import engine as E, tables, workloads as W  # noqa: E402
import node_score_fast as NF  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, _, watts = q.stdout.strip().partition(",") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit_w": float(watts) if watts.strip() else None}


def churn_input():
    rng = W.SplitMix64(5)
    sizes = (rng.next(20000) % np.uint64(16) + np.uint64(1)).astype(np.int64)
    sizes = sizes[:int(np.searchsorted(np.cumsum(sizes), 65536)) + 1]
    sizes[-1] -= int(sizes.sum()) - 65536
    node_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    bits = rng.next(65536 * 8).reshape(65536, 8) >> np.uint64(63)
    occ = (bits.astype(np.uint8) << np.arange(8, dtype=np.uint8)).sum(axis=1).astype(np.uint8)
    frees = np.zeros(2000, dtype=E.REQUEST_DTYPE)
    frees["handle"] = (rng.next(2000) % np.uint64(65536)).astype(np.uint32)
    frees["op"], frees["start"], frees["size"] = E.OP_FREE, (rng.next(2000) % np.uint64(7)).astype(np.uint8), 1
    req = np.concatenate([frees, W.alloc_requests(W.mix_profiles(rng, 20000))])
    return node_off, occ, E.make_profiles(tables.H100_80GB), req


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = card()
    stream = torch.cuda.Stream()
    lines = []
    inputs = {"c3": W.config3(), "churn": churn_input()}
    for name, (node_off, occ, rows, req) in inputs.items():
        G = int(node_off[-1])
        for policy, label in ((E.POLICY_MOST_ALLOCATED, "most_allocated"), (E.POLICY_LEAST_ALLOCATED, "least_allocated"),
                              (E.POLICY_BEST_FIT, "best_fit")):
            eng = E.Engine(max_gpus=max(4096, G), max_batch=len(req), policy=policy)
            eng.set_stream(stream.cuda_stream)
            eng.load_profiles(rows)
            ev, host = [], []
            for rep in range(args.reps + 1):            # the first call sizes the buffers and is not counted
                eng.load_inventory(node_off, occ)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(stream)
                out = eng.place_batch(req)
                e1.record(stream)
                t1 = time.perf_counter()
                e1.synchronize()
                if rep:
                    ev.append(e0.elapsed_time(e1))
                    host.append((t1 - t0) * 1e3)
            t0 = time.process_time()
            if policy == E.POLICY_BEST_FIT:
                ref = oracle.Fast(node_off, rows, policy=E.POLICY_BEST_FIT)
                ref.load(occ)
                want = ref.place(req)
                after = ref.occupancy()
            else:
                want, after = NF.place(node_off, rows, occ, req, policy)
            cpu_ms = (time.process_time() - t0) * 1e3
            assert np.array_equal(out, want) and np.array_equal(eng.read_occupancy(), after), (name, label)
            line = {"input": name, "policy": label, "gpus": G, "nodes": len(node_off) - 1, "requests": len(req),
                    "placed": int((out["status"] == E.ST_PLACED).sum()), "ms_events": round(float(np.median(ev)), 3),
                    "ms_host": round(float(np.median(host)), 3), "checker_one_core_ms": round(cpu_ms, 1),
                    "checker": "oracle ref_fast" if policy == E.POLICY_BEST_FIT else "node_score_fast", "identical_to_checker": True, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
            eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
