"""Times gang preemption (isl_preempt on an ISL_FLAG_GANG_PREEMPT engine, k_preempt_gangs) on the config-4 inventory: 65 536 GPUs
(8 192 nodes x 8) pre-filled to 50 % by workloads.Churn, then filled with C3-mix pods until a gang of eight 1g pods no longer fits
without evictions on any locality.  Every live allocation is listed as a victim with a SplitMix64 rank 0-7; the gangs, of 1-8 pods of
the C3 mix, run at rank 8.  At 50 % alone (DESIGN.md 4.7's input) no gang would evict anything.

For 1, 64 and 1 024 gangs per locality (any node, one node, distinct nodes): the flagged call's time from CUDA events and from the host
clock (medians), the unflagged isl_preempt on the same requests flattened into pods, and the brute force of tests/gang_preempt_fast.cpp
on one CPU core.  A line is printed only after the flagged call's records and evict rows were found byte-identical to the brute force
and the unflagged call's to tests/preempt_fast.cpp.  The card and its power limit are read in the same run.

    python tools/gang_preempt_time.py [--reps 7] [--out results/gang_preempt_time.json]
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
import gang_preempt_fast as GF  # noqa: E402
import preempt_fast as PF  # noqa: E402

LOCALITIES = {"any_node": (E.GANG_ANY_NODES, 0), "one_node": (E.GANG_ONE_NODE, E.FLAG_GANG_ONE_NODE),
              "distinct_nodes": (E.GANG_DISTINCT_NODES, E.FLAG_GANG_DISTINCT_NODES)}


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True)
    name, _, watts = q.stdout.strip().partition(",") if q.returncode == 0 else (torch.cuda.get_device_name(0), "", "")
    return {"gpu": name.strip(), "power_limit_w": float(watts) if watts.strip() else None}


def filled_cluster():
    """The config-4 inventory at 50 % (Churn), then C3-mix pods placed first-fit in batches until a batch places under 1 %."""
    churn = W.Churn(n_nodes=8192, gpus_per_node=8, n_ops=0, fill=0.5)
    ref = oracle.Fast(churn.node_off, churn.rows)
    ref.load(np.zeros(churn.G, dtype=np.uint8))
    churn.generate(ref.place)
    live = churn._live
    gpu, start, size = [churn._gpu[:live]], [churn._start[:live]], [churn._size[:live]]
    rng = W.SplitMix64(3)
    while True:
        res = ref.place(W.alloc_requests(W.mix_profiles(rng, 4096)))
        ok = res[res["status"] == E.ST_PLACED]
        gpu.append(ok["gpu"]); start.append(ok["start"]); size.append(ok["size"])
        if len(ok) < 41:
            break
    vic = np.zeros(sum(len(g) for g in gpu), dtype=E.VICTIM_DTYPE)
    vic["gpu"], vic["start"], vic["size"] = np.concatenate(gpu), np.concatenate(start), np.concatenate(size)
    vic["priority"] = (W.SplitMix64(7).next(len(vic)) % np.uint64(8)).astype(np.uint8)
    return churn, ref.occupancy(), vic


def gangs(rng, n_gangs, rows):
    """n_gangs gangs of 1-8 pods of the C3 mix, handle = gang index, all at rank 8."""
    sizes = (rng.next(n_gangs) % np.uint64(8)).astype(np.int64) + 1
    req = W.alloc_requests(W.mix_profiles(rng, int(sizes.sum())))
    req["handle"] = np.repeat(np.arange(n_gangs), sizes).astype(np.uint32)
    return req, np.full(len(req), 8, dtype=np.uint8)


def timed(eng, stream, reps, *args):
    eng.preempt(*args)                                  # warm-up: buffers sized, modules loaded
    ev, host = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        out = eng.preempt(*args)
        e1.record(stream)
        t1 = time.perf_counter()
        e1.synchronize()
        ev.append(e0.elapsed_time(e1))
        host.append((t1 - t0) * 1e3)
    return out, round(float(np.median(ev)), 4), round(float(np.median(host)), 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    churn, occ, vic = filled_cluster()
    info = card()
    names = list(range(churn.rows.shape[0]))
    one_g = np.zeros(8, dtype=E.REQUEST_DTYPE)
    one_g["profile"] = names[0]                         # the first row of the H100 table: 1g.10gb
    full = {}
    for name, (loc, _f) in LOCALITIES.items():          # the fill: no 1g gang of eight fits without evicting
        _rc, o, _e = GF.preempt(churn.node_off, churn.rows, occ, one_g, np.zeros(8, dtype=np.uint8), vic[:0], locality=loc)
        full[name] = bool((o["status"] != E.ST_PLACED).all())
    stream = torch.cuda.Stream()
    plain = E.Engine(max_gpus=churn.G, max_batch=8192)
    plain.set_stream(stream.cuda_stream)
    plain.load_profiles(churn.rows)
    plain.load_inventory(churn.node_off, occ)
    lines = []
    for name, (loc, flag) in LOCALITIES.items():
        eng = E.Engine(max_gpus=churn.G, max_batch=8192, flags=E.FLAG_GANG_PREEMPT | flag)
        eng.set_stream(stream.cuda_stream)
        eng.load_profiles(churn.rows)
        eng.load_inventory(churn.node_off, occ)
        rng = W.SplitMix64(11)
        for n_gangs in (1, 64, 1024):
            req, prio = gangs(rng, n_gangs, churn.rows)
            (out, evict), ms_ev, ms_host = timed(eng, stream, args.reps, req, prio, vic)
            t0 = time.process_time()
            rc, want, want_ev = GF.preempt(churn.node_off, churn.rows, occ, req, prio, vic, locality=loc)
            cpu_ms = (time.process_time() - t0) * 1e3
            assert rc == E.OK and np.array_equal(out, want) and np.array_equal(evict, want_ev), (name, n_gangs)
            pods = req.copy()
            pods["handle"] = np.arange(len(pods))
            (p_out, p_evict), p_ev, _p_host = timed(plain, stream, args.reps, pods, prio, vic)
            rc, p_want, p_want_ev = PF.preempt(churn.node_off, churn.rows, occ, pods, prio, vic)
            assert rc == E.OK and np.array_equal(p_out, p_want) and np.array_equal(p_evict, p_want_ev), (name, n_gangs)
            assert np.array_equal(eng.read_occupancy(), occ)
            committed = sum(1 for g in range(n_gangs) if (out["status"][req["handle"] == g] == E.ST_PLACED).all())
            line = {"locality": name, "gangs": n_gangs, "pods": len(req), "gpus": churn.G, "victims": len(vic),
                    "full_for_8x1g": full[name], "committed": committed, "evicting_pods": int((evict != E.GPU_NONE).any(axis=1).sum()),
                    "ms_events": ms_ev, "ms_host": ms_host, "unflagged_ms_events": p_ev, "cpu_one_core_ms": round(cpu_ms, 2),
                    "identical_to_checker": True, **info}
            print(json.dumps(line), flush=True)
            lines.append(line)
        eng.close()
    plain.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
