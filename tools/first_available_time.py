"""Times profile alternatives (ISL_FLAG_FIRST_AVAILABLE, k_bestfit's and k_nodefit's pod loops) against what a caller has without them.

Inputs (each pod lists its profile, then the next two smaller profiles of the H100-80GB table, largest first):
  c3     BASELINE config 3: 100 000 pods of the H100 mix (seed 42) on 512 empty 8-GPU nodes (4 096 GPUs)
  half   65 536 GPUs in 8-GPU nodes, every slice busy with probability 1/2 (SplitMix64 seed 5), 20 000 pods of the H100 mix

For each input and policy (FIRST_FIT, BEST_FIT, MOST_ALLOCATED):
  flagged   one isl_place_batch of every pod's alternatives on a flagged engine
  first     one isl_place_batch of the first choices only on the unflagged engine (FIRST_FIT: the segment pipeline)
  emulated  the per-pod emulation on the unflagged engine for the first --prefix pods: one synchronous isl_place_batch per alternative
            until one places; its records are checked against the flagged engine's on the same prefix
Times are medians of --reps calls (CUDA events and host clock, the inventory reloaded before each); the flagged records and final
occupancy are checked byte for byte against the brute force of tests/first_available_fast.cpp, whose one-core time is printed beside.
A line is printed only after its checks passed.  Last, the latency of a one-pod flagged call (three alternatives) on each engine.
The card and its power limit are read in the same run.

    python tools/first_available_time.py [--reps 5] [--prefix 500] [--out results/first_available_time.json]
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
import first_available_fast as F  # noqa: E402

POLICIES = ((E.POLICY_FIRST_FIT, "first_fit"), (E.POLICY_BEST_FIT, "best_fit"), (E.POLICY_MOST_ALLOCATED, "most_allocated"))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, _, watts = q.stdout.strip().partition(",") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit_w": float(watts) if watts.strip() else None}


def with_fallbacks(first):
    """Every pod's profile, then the next two smaller profiles (by slices, table order among equals), as one run per pod."""
    size = np.array([r[1] for r in tables.H100_80GB])
    order = sorted(range(len(size)), key=lambda p: (-size[p], p))
    out = []
    for i, p in enumerate(first):
        k = order.index(int(p))
        smaller = [q for q in order[k + 1:] if size[q] < size[p]][:2]
        out += [(i, q, E.OP_ALLOC, 0, 0) for q in [int(p)] + smaller]
    return np.array(out, dtype=E.REQUEST_DTYPE)


def half_input():
    rng = W.SplitMix64(5)
    G = 65536
    bits = rng.next(G * 8).reshape(G, 8) >> np.uint64(63)
    occ = (bits.astype(np.uint8) << np.arange(8, dtype=np.uint8)).sum(axis=1).astype(np.uint8)
    return W.node_offsets(G // 8, 8), occ, E.make_profiles(tables.H100_80GB), W.alloc_requests(W.mix_profiles(rng, 20000))


def timed(eng, stream, node_off, occ, req, reps):
    ev, host = [], []
    for rep in range(reps + 1):                 # the first call sizes the buffers and is not counted
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
    return out, round(float(np.median(ev)), 3), round(float(np.median(host)), 3)


def make(policy, G, batch, flags, stream, rows):
    eng = E.Engine(max_gpus=max(4096, G), max_batch=batch, policy=policy, flags=flags)
    eng.set_stream(stream.cuda_stream)
    eng.load_profiles(rows)
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--prefix", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = card()
    stream = torch.cuda.Stream()
    lines = []
    for name, (node_off, occ, rows, first) in {"c3": W.config3(), "half": half_input()}.items():
        G = int(node_off[-1])
        req = with_fallbacks(first["profile"])
        for policy, label in POLICIES:
            flagged = make(policy, G, len(req), E.FLAG_FIRST_AVAILABLE, stream, rows)
            plain = make(policy, G, len(req), 0, stream, rows)
            out, ms_ev, ms_host = timed(flagged, stream, node_off, occ, req, args.reps)
            t0 = time.process_time()
            want, after, placed = F.place(node_off, rows, occ, req, policy, E.QUIRKS_REF_EXACT)
            cpu_ms = (time.process_time() - t0) * 1e3
            assert np.array_equal(out, want) and np.array_equal(flagged.read_occupancy(), after), (name, label)
            first_out, first_ev, first_host = timed(plain, stream, node_off, occ, first, args.reps)
            # the per-pod emulation on the first --prefix pods, against the flagged engine on the same prefix
            pre = req[req["handle"] < args.prefix]
            flagged.load_inventory(node_off, occ)
            want_pre = flagged.place_batch(pre)
            plain.load_inventory(node_off, occ)
            torch.cuda.synchronize()
            got_pre = np.zeros(len(pre), dtype=E.RESULT_DTYPE)
            t0 = time.perf_counter()
            done = -1
            for i in range(len(pre)):
                pod = int(pre["handle"][i])
                if pod == done:
                    got_pre[i] = (E.GPU_NONE, E.START_NONE, rows[pre["profile"][i]]["size"], E.ST_ALT_SKIPPED)
                    continue
                got_pre[i] = plain.place_batch(pre[i:i + 1])[0]
                if got_pre[i]["status"] == E.ST_PLACED:
                    done = pod
            emu_ms = (time.perf_counter() - t0) * 1e3
            assert np.array_equal(got_pre, want_pre), (name, label, "emulation")
            line = {"input": name, "policy": label, "gpus": G, "pods": len(first), "requests": len(req), "placed_pods": placed,
                    "placed_first_choice_only": int((first_out["status"] == E.ST_PLACED).sum()),
                    "flagged_ms_events": ms_ev, "flagged_ms_host": ms_host, "first_choices_ms_events": first_ev,
                    "first_choices_ms_host": first_host, "emulated_pods": args.prefix, "emulated_ms_host": round(emu_ms, 1),
                    "emulated_us_per_pod": round(emu_ms * 1e3 / args.prefix, 1), "brute_force_one_core_ms": round(cpu_ms, 1),
                    "identical_to_brute_force": True, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
            flagged.close()
            plain.close()
    one = np.array([(0, 5, E.OP_ALLOC, 0, 0), (0, 2, E.OP_ALLOC, 0, 0), (0, 0, E.OP_ALLOC, 0, 0)], dtype=E.REQUEST_DTYPE)   # 7g, 2g, 1g
    node_off, occ = W.node_offsets(512, 8), np.full(4096, 0x0F, dtype=np.uint8)
    for policy, label in POLICIES:
        eng = make(policy, 4096, 1024, E.FLAG_FIRST_AVAILABLE, stream, E.make_profiles(tables.H100_80GB))
        eng.load_inventory(node_off, occ)
        host = []
        for rep in range(201):
            t0 = time.perf_counter()
            out = eng.place_batch(one)
            if rep:
                host.append((time.perf_counter() - t0) * 1e6)
            eng.load_inventory(node_off, occ)
        assert [int(s) for s in out["status"]] == [E.ST_NO_CAPACITY, E.ST_PLACED, E.ST_ALT_SKIPPED]
        line = {"input": "one_pod", "policy": label, "gpus": 4096, "requests": 3, "flagged_us_host_median": round(float(np.median(host)), 1),
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
