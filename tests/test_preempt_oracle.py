"""isl_preempt's two CPU restatements (tests/preempt_fast.cpp on flat bytes, tests/preempt_oracle.py on custom-resource dicts): the
hand-derived known answers, agreement on random clusters, and the consequences of rule 5 the header states."""
import random

import numpy as np
import pytest

import oracle
from instaslice_b200 import engine as E
from instaslice_b200 import tables

import preempt_fast as PF
import preempt_oracle as PO


def run_fast(case_or_inputs):
    node_off, rows, node_table, occ, req, prio, vic, quirks, policy = case_or_inputs
    return PF.preempt(node_off, rows, occ, req, prio, vic, quirks=quirks, policy=policy, node_table=node_table)


@pytest.mark.parametrize("case", PO.kat_cases(), ids=lambda c: c["name"])
def test_kat_fast(case):
    rc, out, evict = run_fast(PO.case_inputs(case))
    recs, ev = PO.expected(case)
    assert rc == E.OK
    assert [tuple(int(x) for x in r) for r in out] == recs
    assert [[int(k) for k in row if k != E.GPU_NONE] for row in evict] == ev
    assert (evict[[r[3] != E.ST_PLACED for r in recs]] == E.GPU_NONE).all()


@pytest.mark.parametrize("case", PO.kat_cases(), ids=lambda c: c["name"])
def test_kat_cr(case):
    items = PO.case_items(case)
    pods = [{"profile": p, "rank": r} for p, r in case["requests"]]
    got = PO.preempt_cr(items, pods, {"v%d" % k: v[3] for k, v in enumerate(case["victims"])}, PO.QUIRKS[case["quirks"]],
                        PO.POLICY[case["policy"]])
    recs, ev = PO.expected(case)
    for (kind, where, gone), r, e in zip(got, recs, ev):
        if r[3] != E.ST_PLACED:
            assert kind == "none"
            continue
        assert kind == ("preempt" if e else "fits")
        assert (int(where["gpuUUID"][4:]), where["start"], where["size"]) == r[:3]
        assert [int(u[1:]) for u in gone] == e


TABLE_NAMES = ["a100-40gb", "h100-80gb", "a30-24gb"]


def random_cluster(rnd, n_gpus):
    """Instaslice objects with random allocations and dangling Prepared slices, a random victim set with random ranks (255 included)."""
    n_nodes = rnd.randint(1, min(n_gpus, 8))
    cuts = sorted(rnd.sample(range(1, n_gpus), n_nodes - 1)) if n_nodes > 1 else []
    node_off = [0] + cuts + [n_gpus]
    tabs = rnd.sample(TABLE_NAMES, 2)
    items, ranks, uid = [], {}, 0
    for n in range(n_nodes):
        t = tabs[rnd.randrange(2)]
        spec = {"MigGPUUUID": {"GPU-%06d" % g: "" for g in range(node_off[n], node_off[n + 1])},
                "migplacement": tables.migplacement(tables.TABLES[t]), "prepared": {}, "allocations": {}}
        for g in range(node_off[n], node_off[n + 1]):
            s = 0
            while s < 8:
                z = rnd.randint(1, min(4, 8 - s))
                kind = rnd.random()
                if kind < 0.55:
                    spec["allocations"]["u%d" % uid] = {"gpuUUID": "GPU-%06d" % g, "start": s, "size": z, "allocationStatus": "created"}
                    if rnd.random() < 0.8:
                        ranks["u%d" % uid] = rnd.choice([rnd.randrange(8), rnd.randrange(256)])
                    uid += 1
                elif kind < 0.62:
                    spec["prepared"]["q%d" % uid] = {"parent": "GPU-%06d" % g, "start": s, "size": z, "podUUID": ""}
                    uid += 1
                s += z
        items.append({"metadata": {"name": "node-%d" % n}, "spec": spec})
    return items, ranks


def flat_inputs(items, ranks, pods, quirks, policy):
    """The same cluster as the engine sees it: canonical GPUs, occupancy bytes, tables, victims ordered by (GPU, start)."""
    table_names, node_table = [], []
    for it in items:
        mig = it["spec"]["migplacement"]
        key = next(k for k, v in tables.TABLES.items() if tables.migplacement(v) == mig)
        if key not in table_names:
            table_names.append(key)
        node_table.append(table_names.index(key))
    names, rows = E.make_profile_tables([tables.TABLES[t] for t in table_names])
    node_off, occ, vic, uids = [0], [], [], []
    for it in items:
        for u in sorted(it["spec"]["MigGPUUUID"]):
            g = len(occ)
            b = 0
            for x in it["spec"]["prepared"].values():
                if x["parent"] == u:
                    b |= PO.span(x["start"], x["size"])
            for k, a in sorted(it["spec"]["allocations"].items(), key=lambda e: e[1]["start"]):
                if a["gpuUUID"] == u:
                    b |= PO.span(a["start"], a["size"])
                    if k in ranks:
                        vic.append((g, a["start"], a["size"], ranks[k], 0))
                        uids.append(k)
            occ.append(b)
        node_off.append(len(occ))
    req = np.zeros(len(pods), dtype=E.REQUEST_DTYPE)
    req["profile"] = [names.index(p["profile"]) if p["profile"] in names else E.PROFILE_UNKNOWN for p in pods]
    req["op"] = E.OP_ALLOC
    return (np.array(node_off, dtype=np.uint32), rows, np.array(node_table, dtype=np.uint8), np.array(occ, dtype=np.uint8), req,
            np.array([p["rank"] for p in pods], dtype=np.uint8), np.array(vic, dtype=E.VICTIM_DTYPE), quirks, policy), uids


def random_pods(rnd, items, n):
    names = sorted({r["profile"] for it in items for r in it["spec"]["migplacement"]}) + ["9g.99gb"]
    return [{"profile": rnd.choice(names), "rank": rnd.choice([rnd.randrange(10), rnd.randrange(256)])} for _ in range(n)]


@pytest.mark.parametrize("seed", range(24))
def test_restatements_agree(seed):
    rnd = random.Random(seed)
    n_gpus = rnd.choice([1, 2, 7, 33, 128, 512])
    items, ranks = random_cluster(rnd, n_gpus)
    quirks = rnd.choice([E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
    policy = rnd.choice([E.POLICY_FIRST_FIT, E.POLICY_RIGHT_TO_LEFT, E.POLICY_BEST_FIT])
    pods = random_pods(rnd, items, rnd.randint(1, 40))
    inputs, uids = flat_inputs(items, ranks, pods, quirks, policy)
    rc, out, evict = run_fast(inputs)
    assert rc == E.OK
    got = PO.preempt_cr(items, pods, ranks, quirks, policy)
    for (kind, where, gone), r, row in zip(got, out, evict):
        gone_fast = [uids[int(k)] for k in row if k != E.GPU_NONE]
        if r["status"] != E.ST_PLACED:
            assert kind == "none" and not gone_fast
            continue
        assert kind == ("preempt" if gone_fast else "fits")
        assert (int(where["gpuUUID"][4:]), where["start"], where["size"]) == (int(r["gpu"]), int(r["start"]), int(r["size"]))
        assert gone == gone_fast


@pytest.mark.parametrize("seed", range(12))
def test_rule5_consequences(seed):
    """(a) the start is what the start search returns with V removed; every victim is below the preemptor; victims leave whole."""
    rnd = random.Random(1000 + seed)
    items, ranks = random_cluster(rnd, rnd.choice([7, 64, 300]))
    quirks = rnd.choice([E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
    pods = random_pods(rnd, items, 30)
    inputs, _uids = flat_inputs(items, ranks, pods, quirks, E.POLICY_FIRST_FIT)
    node_off, rows, node_table, occ, req, prio, vic, _q, _p = inputs
    rc, out, evict = run_fast(inputs)
    assert rc == E.OK
    gtab = np.repeat(node_table, np.diff(node_off))
    occ = occ.copy()
    for i, (r, row) in enumerate(zip(out, evict)):
        if r["status"] != E.ST_PLACED:
            assert (row == E.GPU_NONE).all()
            continue
        g = int(r["gpu"])
        ks = [int(k) for k in row if k != E.GPU_NONE]
        assert ks == sorted(ks)
        for k in ks:
            assert int(vic[k]["gpu"]) == g and int(vic[k]["priority"]) < int(prio[i])
            occ[g] &= ~np.uint8(PO.span(vic[k]["start"], vic[k]["size"]))
        assert oracle.start_for(rows[gtab[g], req[i]["profile"]], quirks, int(occ[g])) == int(r["start"])
        occ[g] |= np.uint8(PO.span(r["start"], r["size"]))


@pytest.mark.parametrize("quirks", [E.QUIRKS_REF_EXACT, E.QUIRKS_FIXED])
def test_no_victims_is_first_fit(quirks):
    rng = np.random.default_rng(5)
    node_off = np.arange(0, 257, 8, dtype=np.uint32)
    occ = (rng.integers(0, 256, 256) & rng.integers(0, 256, 256)).astype(np.uint8)
    rows = E.make_profiles(tables.H100_80GB)
    req = np.zeros(300, dtype=E.REQUEST_DTYPE)
    req["profile"] = rng.integers(0, len(rows), 300)
    rc, out, evict = PF.preempt(node_off, rows, occ, req, np.full(300, 200, dtype=np.uint8), np.zeros(0, dtype=E.VICTIM_DTYPE), quirks=quirks)
    assert rc == E.OK and (evict == E.GPU_NONE).all()
    ref = oracle.Fast(node_off, rows, quirks=quirks)
    ref.load(occ)
    want = np.concatenate([ref.place(req[i:i + 1]) for i in range(len(req))])
    assert np.array_equal(out, want)


def test_checker_rejects_malformed_victims():
    node_off = np.array([0, 1], dtype=np.uint32)
    rows = E.make_profiles(tables.A100_40GB)
    req = np.zeros(1, dtype=E.REQUEST_DTYPE)
    for v in [(0, 0, 0, 1, 0), (0, 6, 3, 1, 0), (1, 0, 1, 1, 0), (0, 7, 1, 1, 0)]:
        rc, _, _ = PF.preempt(node_off, rows, np.array([0x0F], np.uint8), req, np.ones(1, np.uint8), np.array([v], dtype=E.VICTIM_DTYPE))
        assert rc == E.EINVAL, v
    overlap = np.array([(0, 0, 2, 1, 0), (0, 1, 1, 1, 0)], dtype=E.VICTIM_DTYPE)
    assert PF.preempt(node_off, rows, np.array([0x0F], np.uint8), req, np.ones(1, np.uint8), overlap)[0] == E.EINVAL
