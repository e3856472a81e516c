"""Times the node-scored few-node, elastic and balanced gangs (isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE |
ISL_FLAG_GANG_NODE_SCORE_ALL engine) against the kernels they extend:

- few nodes: k_ganglocal<few_nodes, node_score> against k_ganglocal<few_nodes> (a FIRST_FIT few-node engine) on DESIGN.md 4.16's
  inventory and gangs (tools/gang_score_time.py: 65 536 GPUs in 7 669 nodes, 4 255 gangs of 2, 4 and 8 pods of the H100 mix);
- elastic: the same gangs with a minimum of half their members (m = k/2) as one-node and few-node bytes, on
  k_ganglocal<per_gang, min_members, node_score>, against the same bytes without a minimum (k_ganglocal<per_gang, node_score>);
- balanced: bytes 4 and 5 (maxSkew 1 and 2) on k_ganglocal<per_gang, node_score, balanced> against k_ganglocal<per_gang, balanced> on a
  FIRST_FIT engine, on DESIGN.md 4.17's inventory and replica gangs of 8, 16 and 32 (tools/gang_balance_time.py).

Every line is printed only after the scored call's records, occupancy and stats.placed were found byte-identical to the brute force of
tests/gang_score_all_fast.cpp.  Times are medians of --reps synchronous calls by CUDA events, the inventory reloaded before each; the
card and its power limit are read in the same run.

    python tools/gang_score_all_time.py [--reps 5] [--out results/gang_score_all_time.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from instaslice_b200 import engine as E, workloads as W  # noqa: E402
import gang_locality_oracle as GLO  # noqa: E402
import gang_score_all_fast as GSA  # noqa: E402
from gang_node_time import prefilled  # noqa: E402
from gang_score_time import card, churn_inventory, gang_call, timed  # noqa: E402

ALL = E.FLAG_GANG_NODE_SCORE | E.FLAG_GANG_NODE_SCORE_ALL
POLICIES = {"most_allocated": E.POLICY_MOST_ALLOCATED, "least_allocated": E.POLICY_LEAST_ALLOCATED}


def engine(policy, flags, rows, G, n, stream):
    eng = E.Engine(max_gpus=G, max_batch=n, policy=policy, flags=flags)
    eng.set_stream(stream.cuda_stream)
    eng.load_profiles(rows)
    return eng


def measured(eng, rows, stream, reps, node_off, occ, req, off, policy, locality, elastic=False):
    """The call's median event time, after its records, occupancy and stats.placed were checked against the brute force."""
    out, ms, _ = timed(eng, stream, reps, node_off, occ, lambda: eng.place_gangs(req, off))
    occ_after, placed = eng.read_occupancy(), eng.stats()["placed"]
    want, occ_want, placed_want = GSA.place_gangs(node_off, rows, occ, req, off, policy, locality, elastic=elastic)
    assert np.array_equal(out, want) and np.array_equal(occ_after, occ_want) and placed == placed_want, (policy, locality, elastic)
    return ms, placed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gang_score_all_time.py measures on a GPU and found none")
    info = card()
    stream = torch.cuda.Stream()
    lines = []

    def emit(line):
        line.update(identical_to_brute_force=True, **info)
        print(json.dumps(line), flush=True)
        lines.append(line)

    node_off, occ, rows = churn_inventory()
    req, off = gang_call()
    G, n, n_gangs = int(node_off[-1]), len(req), len(off) - 1
    sizes = np.diff(off.astype(np.int64))
    ff = engine(E.POLICY_FIRST_FIT, E.FLAG_GANG_FEW_NODES, rows, G, n, stream)
    _, ff_ms, _ = timed(ff, stream, args.reps, node_off, occ, lambda: ff.place_gangs(req, off))
    ff.close()
    half = req.copy()
    alloc = half["op"] == E.OP_ALLOC
    half["size"][alloc] = np.repeat(sizes // 2, sizes)[alloc]
    for pname, policy in POLICIES.items():
        eng = engine(policy, ALL | E.FLAG_GANG_FEW_NODES, rows, G, n, stream)
        ms, placed = measured(eng, rows, stream, args.reps, node_off, occ, req, off, policy, E.GANG_FEW_NODES)
        eng.close()
        emit({"what": "few_nodes", "policy": pname, "gangs": n_gangs, "pods": n, "gpus": G, "nodes": len(node_off) - 1, "placed": placed,
              "scored_ms_events": ms, "first_fit_few_nodes_ms_events": ff_ms, "scored_over_first_fit": round(ms / ff_ms, 3),
              "us_per_gang": round(ms * 1e3 / n_gangs, 2)})
        el = engine(policy, ALL | E.FLAG_GANG_LOCALITY | E.FLAG_GANG_MIN_MEMBERS, rows, G, n, stream)
        plain = engine(policy, ALL | E.FLAG_GANG_LOCALITY, rows, G, n, stream)
        for byte, bname in ((E.GANG_ONE_NODE, "one_node"), (E.GANG_FEW_NODES, "few_nodes")):
            r_el = GLO.with_locality(half, off, np.full(n_gangs, byte))
            r_plain = GLO.with_locality(req, off, np.full(n_gangs, byte))
            ms_el, placed_el = measured(el, rows, stream, args.reps, node_off, occ, r_el, off, policy, GSA.PER_GANG, elastic=True)
            ms_plain, placed_plain = measured(plain, rows, stream, args.reps, node_off, occ, r_plain, off, policy, GSA.PER_GANG)
            emit({"what": "elastic_" + bname, "policy": pname, "gangs": n_gangs, "pods": n, "min_members": "k/2", "placed": placed_el,
                  "placed_without_minimum": placed_plain, "elastic_ms_events": ms_el, "without_minimum_ms_events": ms_plain,
                  "elastic_over_without": round(ms_el / ms_plain, 3)})
        el.close()
        plain.close()

    rng = W.SplitMix64(42)                                  # tools/gang_balance_time.py's inventory and replica gangs
    node_off = W.node_offsets(8192, 8)
    rows = E.make_profiles(W.tables.H100_80GB)
    occ = prefilled(node_off, rows, rng)
    pods = 4096
    mix = W.mix_profiles(rng, pods)
    G = int(node_off[-1])
    unscored = engine(E.POLICY_FIRST_FIT, E.FLAG_GANG_LOCALITY | E.FLAG_GANG_BALANCED, rows, G, pods, stream)
    scored = {p: engine(policy, ALL | E.FLAG_GANG_LOCALITY | E.FLAG_GANG_BALANCED, rows, G, pods, stream) for p, policy in POLICIES.items()}
    for k in (8, 16, 32):
        base = W.alloc_requests(np.repeat(mix[::k], k)[:pods])
        off = np.r_[np.arange(0, len(base), k), len(base)].astype(np.uint32)
        for skew in (1, 2):
            req = GLO.with_locality(base, off, np.full(len(off) - 1, E.gang_balanced_nodes(skew)))
            _, ms_ff, _ = timed(unscored, stream, args.reps, node_off, occ, lambda: unscored.place_gangs(req, off))
            for pname, policy in POLICIES.items():
                ms, placed = measured(scored[pname], rows, stream, args.reps, node_off, occ, req, off, policy, GSA.PER_GANG)
                emit({"what": "balanced", "policy": pname, "gang_size": k, "max_skew": skew, "gangs": len(off) - 1, "pods": len(base),
                      "gpus": G, "nodes": len(node_off) - 1, "placed": placed, "scored_ms_events": ms, "first_fit_ms_events": ms_ff,
                      "scored_over_first_fit": round(ms / ms_ff, 3), "us_per_member": round(ms * 1e3 / len(base), 3)})
    unscored.close()
    for eng in scored.values():
        eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
