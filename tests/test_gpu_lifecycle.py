"""One long-lived engine whose state moves between calls, as the controller, the host mirror and the Go shim use it: every C-ABI symbol
in every engine state (tests/engine_contract.py), open streams in each of their sub-states, table reloads after a node map, and a random
walk over the whole ABI.  After every call the return code must be the contract's, and after every successful one the records and the
WHOLE occupancy must equal ``engine_contract.Model``'s.  Needs an H100.

The open-stream probes run in a safe order: (i) opened, not launched, and (ii) every batch submitted and waited, have no kernel resident,
so a missing guard shows up as OK instead of ESTATE; (iii) launched with batches still due runs only after (i) and (ii) passed.
"""
import ctypes as C

import numpy as np
import pytest

from instaslice_b200 import engine as E
from instaslice_b200 import tables
from instaslice_b200 import workloads as W

import engine_contract as K
from range_oracle import mixed_requests
from test_gpu_ranges import check_path, delta

pytestmark = pytest.mark.gpu
MIX = [tables.A100_40GB, tables.H100_80GB, tables.A30_24GB]      # table 0 (A100) lacks every H100 and A30 name
MAX_BATCH = 4 * 65536
# symbols the open-stream probes saw refused in sub-states (i) and (ii): the only ones the random walk calls while a kernel is resident
VERIFIED_REFUSED = set()


def table_rows(n_tables):
    """1: the H100 table (isl_load_profiles); 2..3: the first n tables of MIX over the union of all three tables' names, so the name
    list (and the request profile indices) stays the same across reloads."""
    if n_tables == 1:
        return E.make_profiles(tables.H100_80GB)
    names, rows = E.make_profile_tables(MIX)
    return rows[:n_tables]


def load_rows(eng, model, rows):
    if rows.ndim == 1:
        rc = eng._lib.isl_load_profiles(eng._h, len(rows), rows.ctypes.data_as(C.c_void_p))
    else:
        rc = eng._lib.isl_load_profile_tables(eng._h, rows.shape[0], rows.shape[1], rows.ctypes.data_as(C.c_void_p))
    assert rc == model.expected("isl_load_profiles"), rc
    if rc == E.OK:
        model.load_profiles(rows)


def unequal_nodes(rng, G, max_nodes=None):
    """Node offsets of G GPUs in nodes of 1..16 GPUs (or at most ``max_nodes`` nodes of very different sizes)."""
    if max_nodes:
        cuts = np.unique(rng.next(max_nodes - 1) % np.uint64(G)).astype(np.int64)
        return np.unique(np.r_[0, cuts, G]).astype(np.uint32)
    sizes = (1 + rng.next(G) % np.uint64(16)).astype(np.int64)
    off = np.r_[0, np.cumsum(sizes)]
    off = off[off < G]
    return np.r_[off, G].astype(np.uint32)


def random_occ(rng, G):
    return ((rng.next(G) & rng.next(G)) & np.uint64(0x7F)).astype(np.uint8)


# ---- probes: one well-formed call of every symbol ----------------------------------------------------------------------------------------
class Probe:
    """Buffers for one well-formed call of every symbol against an engine and its model.  ``call(name)`` returns the code, or the value
    for a getter."""

    N = 8

    def __init__(self, eng, model):
        import torch
        self.eng, self.lib, self.m = eng, eng._lib, model
        self.req = W.alloc_requests(np.zeros(self.N, dtype=np.uint8))
        self.out = np.zeros(self.N, dtype=E.RESULT_DTYPE)
        self.pin_in, self.pin_out = E.PinnedArray(self.N, E.REQUEST_DTYPE), E.PinnedArray(self.N, E.RESULT_DTYPE)
        self.pin_in.array[:] = self.req
        self.d_in = torch.from_numpy(self.req.view(np.uint8).copy()).cuda()
        self.d_out = torch.zeros(self.N * 8, dtype=torch.uint8, device="cuda")
        self.d_heads = torch.zeros(16 * 4, dtype=torch.uint8, device="cuda")
        self.sizes = np.array([self.N], dtype=np.uint32)
        self.gang_off = np.array([0, self.N], dtype=np.uint32)
        self.prio, self.evict = np.full(self.N, 3, dtype=np.uint8), np.zeros((self.N, 8), dtype=np.uint32)
        self.cap = np.zeros(E.MAX_PROFILES, dtype=np.uint64)
        self.cap2 = np.zeros(E.MAX_PROFILES, dtype=np.uint64)
        self.h64 = C.create_string_buffer(64)
        self.span = np.array([(0, 0, 1, 0)], dtype=E.SPAN_DTYPE)
        self.bytes = np.arange(4, dtype=np.uint8)
        self.ticket = 0
        torch.cuda.synchronize()

    def close(self):
        self.pin_in.free(); self.pin_out.free()

    def call(self, name):
        L, h, m, p = self.lib, self.eng._h, self.m, lambda a: a.ctypes.data_as(C.c_void_p)
        G = max(1, m.G)
        n_nodes = 1 if m.node_off is None else len(m.node_off) - 1
        if name == "isl_create":
            cfg = E.Config(E.ABI_VERSION, 0, 3, -1, 64, 64, 0, 0)
            h2 = C.c_void_p()
            rc = L.isl_create(C.byref(cfg), C.byref(h2))
            L.isl_destroy(h2)
            return rc
        if name == "isl_destroy":
            raise AssertionError("probed on its own engine")
        rows = m.rows if m.rows is not None else table_rows(1)
        occ = m.occ if m.occ is not None else np.zeros(1, dtype=np.uint8)
        node_off = m.node_off if m.node_off is not None else np.array([0, 1], dtype=np.uint32)
        byte = np.array([occ[0] ^ 0x80], dtype=np.uint8)
        tab = np.zeros(n_nodes, dtype=np.uint8)
        d_in, d_out = C.c_void_p(self.d_in.data_ptr()), C.c_void_p(self.d_out.data_ptr())
        calls = {
            "isl_set_stream": lambda: L.isl_set_stream(h, None),
            "isl_synchronize": lambda: L.isl_synchronize(h),
            "isl_load_profiles": lambda: L.isl_load_profiles(h, len(table_rows(1)), p(table_rows(1))),
            "isl_load_profile_tables": lambda: L.isl_load_profile_tables(h, 2, table_rows(2).shape[1], p(table_rows(2))),
            "isl_set_node_tables": lambda: L.isl_set_node_tables(h, n_nodes, p(tab)),
            "isl_load_inventory": lambda: L.isl_load_inventory(h, len(node_off) - 1, p(node_off), p(occ)),
            "isl_read_occupancy": lambda: L.isl_read_occupancy(h, p(np.zeros(G, dtype=np.uint8))),
            "isl_write_occupancy": lambda: L.isl_write_occupancy(h, 0, 1, p(byte)),
            "isl_snapshot_occupancy": lambda: L.isl_snapshot_occupancy(h),
            "isl_restore_occupancy": lambda: L.isl_restore_occupancy(h),
            "isl_num_gpus": lambda: L.isl_num_gpus(h),
            "isl_gpu_to_node": lambda: L.isl_gpu_to_node(h, 0),
            "isl_place_batch": lambda: L.isl_place_batch(h, self.N, p(self.req), p(self.out)),
            "isl_place_batch_device": lambda: L.isl_place_batch_device(h, self.N, d_in, d_out),
            "isl_place_stream": lambda: L.isl_place_stream(h, 1, p(self.sizes), p(self.req), p(self.out)),
            "isl_place_stream_device": lambda: L.isl_place_stream_device(h, 1, p(self.sizes), d_in, d_out),
            "isl_place_batch_range": lambda: L.isl_place_batch_range(h, 0, m.G, self.N, p(self.req), p(self.out)),
            "isl_place_gangs": lambda: L.isl_place_gangs(h, 1, p(self.gang_off), p(self.req), p(self.out)),
            "isl_preempt": lambda: L.isl_preempt(h, self.N, p(self.req), p(self.prio), 0, None, p(self.out), p(self.evict)),
            "isl_free_batch": lambda: L.isl_free_batch(h, 1, p(self.span)),
            "isl_eval_starts": lambda: L.isl_eval_starts(h, 0, 4, p(self.bytes), p(np.zeros(4, dtype=np.uint8))),
            "isl_set_partition": lambda: L.isl_set_partition(h, 0, m.G),
            "isl_place_batch_partitioned": lambda: L.isl_place_batch_partitioned(h, self.N, d_in, d_out, None, C.c_void_p(self.d_heads.data_ptr())),
            "isl_ipc_inbox_handle": lambda: L.isl_ipc_inbox_handle(h, self.h64),
            "isl_ipc_connect": lambda: L.isl_ipc_connect(h, None, 0),
            "isl_connect_local": lambda: L.isl_connect_local(h, None, 0),
            "isl_place_stream_partitioned": lambda: L.isl_place_stream_partitioned(h, 1, p(self.sizes), d_in, d_out, 1),
            "isl_device_occupancy": lambda: L.isl_device_occupancy(h),
            "isl_get_stats": lambda: L.isl_get_stats(h, C.byref(E.Stats())),
            "isl_read_trace": lambda: L.isl_read_trace(h, None, 0, C.byref(C.c_uint32()), C.byref(C.c_uint32())),
            "isl_reset_stats": lambda: L.isl_reset_stats(h),
            "isl_strerror": lambda: L.isl_strerror(E.ESTATE),
            "isl_last_cuda_error": lambda: L.isl_last_cuda_error(h),
            "isl_abi_version": lambda: L.isl_abi_version(),
            "isl_stream_open": lambda: L.isl_stream_open(h, 2),
            "isl_stream_submit": lambda: L.isl_stream_submit(h, self.N, C.c_void_p(self.pin_in.ptr), C.c_void_p(self.pin_out.ptr), None),
            "isl_stream_wait": lambda: L.isl_stream_wait(h, self.ticket),
            "isl_stream_close": lambda: L.isl_stream_close(h),
            "isl_set_causal_window": lambda: L.isl_set_causal_window(h, 0),
            "isl_set_speculation": lambda: L.isl_set_speculation(h, E.SPEC_AUTO),
            "isl_ipc_spec_handle": lambda: L.isl_ipc_spec_handle(h, self.h64),
            "isl_ipc_connect_spec": lambda: L.isl_ipc_connect_spec(h, 0, 0, None, None),
            "isl_connect_spec_local": lambda: L.isl_connect_spec_local(h, 0, 0, None, None),
            "isl_host_alloc": lambda: L.isl_host_free(L.isl_host_alloc(64)),
            "isl_host_free": lambda: L.isl_host_free(None),
            "isl_device_results": lambda: L.isl_device_results(h),
            "isl_ipc_results_handle": lambda: L.isl_ipc_results_handle(h, self.h64),
            "isl_ipc_connect_owner": lambda: L.isl_ipc_connect_owner(h, None),
            "isl_connect_owner_local": lambda: L.isl_connect_owner_local(h, None),
            "isl_set_ring_world": lambda: L.isl_set_ring_world(h, 0),
            "isl_capacity": lambda: L.isl_capacity(h, p(self.cap)),
            "isl_what_if": lambda: L.isl_what_if(h, self.N, p(self.req), p(self.out), p(self.cap), p(self.cap2)),
        }
        return calls[name]()


def refused_probe(eng, model, probe, names, what):
    """Call every symbol in ``names`` that the contract refuses in the model's state; return the first mismatch or None."""
    for name in names:
        want = model.expected(name)
        if want in (K.VALUE, E.OK) or name in ("isl_create", "isl_destroy"):
            continue
        got = probe.call(name)
        if got != want:
            return (what, model.state(), name, "got", got, "want", want)
    return None


def check_getters(eng, model, what):
    assert eng.num_gpus == model.G, what
    if model.G:
        assert eng.gpu_to_node(model.G - 1) == len(model.node_off) - 2, what
    assert eng.gpu_to_node(model.G) == E.GPU_NONE, what
    assert eng.device_occupancy() and eng.device_results(), what
    assert eng._lib.isl_abi_version() == E.ABI_VERSION and eng._lib.isl_strerror(E.ESTATE)


def compare(got, want, eng, model, what):
    bad = np.flatnonzero(got != want)
    assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])
    occ = eng.read_occupancy()
    diff = np.flatnonzero(occ != model.occ)
    assert len(diff) == 0, (what, "occupancy", diff[:5], occ[diff[:5]], model.occ[diff[:5]])


# ---- 1. readiness states -------------------------------------------------------------------------------------------------------------
def engine_in(state, policy, flags, rows, node_off, occ):
    eng = E.Engine(max_gpus=4096, max_batch=MAX_BATCH, policy=policy, flags=flags)
    model = K.Model(policy, E.QUIRKS_REF_EXACT, flags)
    if state in ("profiles", "ready"):
        load_rows(eng, model, rows)
    if state in ("inventory", "ready"):
        eng.load_inventory(node_off, occ)
        model.load_inventory(node_off, occ)
    return eng, model


@pytest.mark.parametrize("policy,flags", [(E.POLICY_FIRST_FIT, 0), (E.POLICY_RIGHT_TO_LEFT, 0), (E.POLICY_BEST_FIT, 0),
                                          (E.POLICY_FIRST_FIT, E.FLAG_ALL_NODES)])
def test_readiness_states(policy, flags):
    """Created, profiles only, inventory only: every symbol returns its contract code.  The refused calls leave nothing behind (the
    getters, the occupancy and the first placement after becoming ready match the model); each accepted one runs on its own engine."""
    rng = W.SplitMix64(11 + policy + flags)
    G = 300
    node_off = unequal_nodes(rng, G, max_nodes=6 if flags else None)
    occ = random_occ(rng, G)
    rows = table_rows(3)
    for state in ("created", "profiles", "inventory"):
        eng, model = engine_in(state, policy, flags, rows, node_off, occ)
        probe = Probe(eng, model)
        miss = refused_probe(eng, model, probe, sorted(K.CODES), state)
        assert miss is None, miss
        check_getters(eng, model, state)
        if model.occ is not None:
            assert np.array_equal(eng.read_occupancy(), model.occ), state
        # the first placement after becoming ready matches the model
        if model.rows is None:
            load_rows(eng, model, rows)
        if model.node_off is None:
            eng.load_inventory(node_off, occ)
            model.load_inventory(node_off, occ)
        req = mixed_requests(rng, model.occ, 0, G, model.n_names, 40)
        compare(eng.place_batch(req), model.place_batch(req), eng, model, (state, "first placement"))
        probe.close()
        eng.close()
        # every call the state accepts, each on a fresh engine in that state
        for name in sorted(K.CODES):
            want = K.expected(name, state, K.Ctx(policy, flags))
            if want != E.OK or name == "isl_destroy":
                continue
            eng, model = engine_in(state, policy, flags, rows, node_off, occ)
            probe = Probe(eng, model)
            assert probe.call(name) == E.OK, (state, name, eng._lib.isl_last_cuda_error(eng._h))
            probe.close()
            assert eng._lib.isl_destroy(eng._h) == E.OK, (state, name)
            eng._h = None


# ---- 2. open streams: every symbol in every sub-state ----------------------------------------------------------------------------------
OPEN_CASES = [("ff-1", E.POLICY_FIRST_FIT, 1, 0), ("rtl-3", E.POLICY_RIGHT_TO_LEFT, 3, 0), ("all-nodes", E.POLICY_FIRST_FIT, 1, E.FLAG_ALL_NODES)]


def open_engine(policy, n_tables, flags, seed, G=4099):
    rng = W.SplitMix64(seed)
    node_off = unequal_nodes(rng, G, max_nodes=5 if flags & E.FLAG_ALL_NODES else None)
    occ = random_occ(rng, G)
    eng = E.Engine(max_gpus=65536, max_batch=MAX_BATCH, policy=policy, flags=flags)
    model = K.Model(policy, E.QUIRKS_REF_EXACT, flags)
    load_rows(eng, model, table_rows(n_tables))
    eng.load_inventory(node_off, occ)
    model.load_inventory(node_off, occ)
    if n_tables > 1:
        nt = (rng.next(len(node_off) - 1) % np.uint64(n_tables)).astype(np.uint8)
        eng.set_node_tables(nt)
        model.set_node_tables(nt)
    return rng, eng, model


@pytest.mark.parametrize("case,policy,n_tables,flags", OPEN_CASES)
def test_open_stream_refuses_every_other_call(case, policy, n_tables, flags):
    rng, eng, model = open_engine(policy, n_tables, flags, 500 + len(case))
    G, mb, n = model.G, 3, 3000
    eng.snapshot_occupancy()                  # a restore that slipped through would revert the stream's commits
    model.snapshot()
    probe = Probe(eng, model)
    names = sorted(set(K.CODES) - K.LEGAL_DURING_OPEN)
    h_in, h_out = E.PinnedArray(mb * n, E.REQUEST_DTYPE), E.PinnedArray(mb * n, E.RESULT_DTYPE)

    def submit(b):
        req = mixed_requests(rng, model.occ, 0, G, model.n_names, n)
        h_in.array[b * n:(b + 1) * n] = req
        t = eng.stream_submit_ptr(n, h_in.ptr + 8 * b * n, h_out.ptr + 8 * b * n)
        model.open[1] += 1
        model.open[2] = True
        eng.stream_wait(t)
        probe.ticket = t
        got, want = h_out.array[b * n:(b + 1) * n].copy(), model.place_stream(req)
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (case, "open batch", b, bad[:5], got[bad[:5]], want[bad[:5]])

    for sub in ("i", "ii", "iii"):
        eng.stream_open(mb)
        model.open = [mb, 0, False]
        miss = None
        try:
            if sub == "ii":
                for b in range(mb):
                    submit(b)
            if sub == "iii":
                submit(0)
            miss = refused_probe(eng, model, probe, names, (case, sub))
            if miss is None and sub == "ii":
                VERIFIED_REFUSED.update(names)
            if miss is None:
                check_getters(eng, model, (case, sub))
                want_submit = model.expected("isl_stream_submit")
                if want_submit != E.OK:         # all batches in: one more is out of range
                    assert probe.call("isl_stream_submit") == want_submit, (case, sub)
                if sub == "i":
                    assert probe.call("isl_stream_wait") == model.expected("isl_stream_wait"), (case, sub)
            if sub == "iii" and miss is None:
                for b in range(1, mb):
                    submit(b)
        finally:
            eng.stream_close()
            model.open = None
        assert miss is None, miss
        # the refused calls changed nothing: the whole occupancy is the model's batch-by-batch answer, the snapshot is still the old one
        assert np.array_equal(eng.read_occupancy(), model.occ), (case, sub)
    eng.restore_occupancy()
    model.restore()
    assert np.array_equal(eng.read_occupancy(), model.occ), (case, "restore after the streams")
    # destroy closes an open stream in every sub-state
    for sub in ("i", "ii", "iii"):
        e2 = E.Engine(max_gpus=65536, max_batch=MAX_BATCH, policy=policy, flags=flags)
        e2.load_profiles(table_rows(1))
        e2.load_inventory(model.node_off, model.occ)
        e2.stream_open(2)
        for b in range({"i": 0, "ii": 2, "iii": 1}[sub]):
            e2.stream_wait(e2.stream_submit_ptr(n, h_in.ptr, h_out.ptr))
        assert e2._lib.isl_destroy(e2._h) == E.OK, sub
        e2._h = None
    h_in.free(); h_out.free()
    probe.close()
    eng.close()


# ---- 3. reloading tables after a node map ------------------------------------------------------------------------------------------
def check_every_path(rng, eng, chunk_eng, bf_eng, model, bf_model, what):
    """k_few, k_small, the chunk path and its scan mode, the plain pipeline, speculative rounds, k_bestfit, capacity, eval_starts and
    what_if against the model; each path's launch count says it ran."""
    G = model.G
    for shape, n in (("few", 8), ("small", 700), ("scan", 5000), ("plain", 6000), ("spec", 6000), ("chunks", 6000), ("mixed", 3000)):
        # "mixed": a host batch that mixes profiles but is too short for the pipeline takes the chunk path
        req = mixed_requests(rng, model.occ, 0, G, model.n_names, n, profile=0 if shape == "scan" else None)
        e = chunk_eng if shape == "chunks" else eng
        if shape == "chunks":
            chunk_eng.write_occupancy(0, model.occ)
        e.set_speculation(E.SPEC_OFF if shape == "plain" else E.SPEC_AUTO)
        before = e.stats()
        got = e.place_batch(req)
        want = model.place_batch(req)
        compare(got, want, e, model, (what, shape))
        check_path(delta(e, before), {"few": "one", "small": "one", "mixed": "chunks"}.get(shape, shape), n, (what, shape), G, 0, G, model.n_tables)
        if shape == "chunks":
            eng.write_occupancy(0, model.occ)
        if shape == "scan":
            # a name table 0 lacks: NO_CAPACITY everywhere once every node is back on table 0, with the default size of the model
            lacking = [p for p in range(model.n_names) if model.sizes()[p] == 0]
            if lacking:
                req = W.alloc_requests(np.full(40, lacking[0], dtype=np.uint8))
                want = model.place_batch(req)
                assert (want["status"] == E.ST_NO_CAPACITY).all()
                compare(eng.place_batch(req), want, eng, model, (what, "lacking name"))
    eng.set_speculation(E.SPEC_AUTO)
    req = mixed_requests(rng, bf_model.occ, 0, G, bf_model.n_names, 1500)
    before = bf_eng.stats()
    compare(bf_eng.place_batch(req), bf_model.place_batch(req), bf_eng, bf_model, (what, "bestfit"))
    check_path(delta(bf_eng, before), "bestfit", 1500, (what, "bestfit"), G, 0, G)
    assert np.array_equal(eng.capacity(), model.capacity()), (what, "capacity")
    for t in range(model.n_tables):
        for p in range(model.n_names):
            occ = np.arange(256, dtype=np.uint8)
            assert np.array_equal(eng.eval_starts(p | t << 8, occ), model.eval_starts(p | t << 8, occ)), (what, "eval_starts", t, p)
    plan = mixed_requests(rng, model.occ, 0, G, model.n_names, 3000)
    got, before_cap, after_cap = eng.what_if(plan)
    want, wb, wa = model.what_if(plan)
    assert np.array_equal(got, want) and np.array_equal(before_cap, wb) and np.array_equal(after_cap, wa), (what, "what_if")
    assert np.array_equal(eng.read_occupancy(), model.occ), (what, "what_if restore")


def test_table_reload_after_node_map():
    """load_inventory -> set_node_tables -> a reload with the same, fewer and more tables, and a single-table isl_load_profiles: the reload
    puts every node back on table 0, and every path agrees with that."""
    rng = W.SplitMix64(4242)
    G = 16000                       # within k_few's 16 384 GPUs
    node_off = W.node_offsets(G // 8, 8)
    occ = random_occ(rng, G)
    engines = [E.Engine(max_gpus=65536, max_batch=MAX_BATCH),
               E.Engine(max_gpus=65536, max_batch=MAX_BATCH, flags=E.FLAG_NO_PIPELINE | E.FLAG_NO_SMALL),
               E.Engine(max_gpus=65536, max_batch=MAX_BATCH, policy=E.POLICY_BEST_FIT)]
    models = [K.Model(), K.Model(), K.Model(E.POLICY_BEST_FIT)]
    for eng, model in zip(engines, models):
        load_rows(eng, model, table_rows(3))
        eng.load_inventory(node_off, occ)
        model.load_inventory(node_off, occ)
    eng, chunk_eng, bf_eng = engines
    model, _, bf_model = models
    for reload in (3, 3, 2, 3, 1):
        nt = (1 + rng.next(len(node_off) - 1) % np.uint64(2)).astype(np.uint8)     # tables 1 and 2 only: table 0 is nobody's
        for e in engines:
            e.set_node_tables(nt)
        model.set_node_tables(nt)
        bf_model.set_node_tables(nt)
        check_every_path(rng, eng, chunk_eng, bf_eng, model, bf_model, ("node map", reload))
        for e in engines:
            rows = table_rows(reload)
            load_rows(e, K.Model(), rows)
        model.load_profiles(table_rows(reload))
        bf_model.load_profiles(table_rows(reload))
        check_every_path(rng, eng, chunk_eng, bf_eng, model, bf_model, ("reload", reload))
        if reload == 1:
            break
        # back to three tables for the next node map
        for e in engines:
            load_rows(e, K.Model(), table_rows(3))
        model.load_profiles(table_rows(3))
        bf_model.load_profiles(table_rows(3))
    for e in engines:
        e.close()


# ---- 4. a random walk over the whole ABI on one long-lived engine -----------------------------------------------------------------
WALK_CASES = [("ff-ref-1", E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT, 1, 0), ("ff-fixed-3", E.POLICY_FIRST_FIT, E.QUIRKS_FIXED, 3, 0),
              ("rtl-3", E.POLICY_RIGHT_TO_LEFT, E.QUIRKS_REF_EXACT, 3, 0), ("bf-fixed", E.POLICY_BEST_FIT, E.QUIRKS_FIXED, 1, 0),
              ("minfrag-3", E.POLICY_MIN_FRAG, E.QUIRKS_REF_EXACT, 3, 0), ("ff-all-nodes", E.POLICY_FIRST_FIT, E.QUIRKS_REF_EXACT, 1, E.FLAG_ALL_NODES)]
N_OPS = 400
GS = (37, 4099, 20000, 65536)
SIZES = (1, 8, 1024, 1025, 5000, 6000, 65537)       # 5000: one profile (scan mode); the others mixed
# the CPU restatements of the best-fit family scan every GPU per request (min-frag also every candidate): requests x GPUs per call
ORACLE_BUDGET = {E.POLICY_BEST_FIT: 4e7, E.POLICY_MIN_FRAG: 3e6}


class Walk:
    def __init__(self, case, policy, quirks, n_tables, flags, seed):
        import torch
        self.case, self.seed, self.n_tables = case, seed, n_tables
        self.rng = W.SplitMix64(seed)
        self.eng = E.Engine(max_gpus=65536, max_batch=MAX_BATCH, policy=policy, quirks=quirks, flags=flags)
        self.m = K.Model(policy, quirks, flags)
        self.probe = Probe(self.eng, self.m)
        self.log = []
        self.torch = torch
        load_rows(self.eng, self.m, table_rows(n_tables))
        self.load_inventory()

    def r(self, k):
        return int(self.rng.next1() % np.uint64(k))

    def note(self, text):
        self.log[-1] += " " + text

    def attempt(self, symbol, fn):
        """Run one engine call; its code must be the contract's.  Returns (ok, result)."""
        want = self.m.expected(symbol)
        try:
            out, rc = fn(), E.OK
        except E.EngineError as err:
            out, rc = None, err.code
        if rc == E.ECUDA:           # never retried: the walk ends here
            raise AssertionError(f"{symbol}: ISL_ECUDA {self.eng._lib.isl_last_cuda_error(self.eng._h).decode()}")
        assert rc == want, (symbol, "got", rc, "want", want)
        self.note(f"rc={rc}")
        return rc == E.OK, out

    def check(self, got, want, what):
        bad = np.flatnonzero(got != want)
        assert len(bad) == 0, (what, bad[:5], got[bad[:5]], want[bad[:5]])

    def check_occupancy(self):
        occ = self.eng.read_occupancy()
        diff = np.flatnonzero(occ != self.m.occ)
        assert len(diff) == 0, ("occupancy", diff[:5], occ[diff[:5]], self.m.occ[diff[:5]])

    # -- draws
    def size(self, cap=None):
        budget = ORACLE_BUDGET.get(self.m.policy)
        ok = [n for n in SIZES if (budget is None or n * self.m.G <= budget or n <= 8) and (cap is None or n <= cap)]
        return ok[self.r(len(ok))]

    def requests(self, n, lo=None, hi=None):
        lo, hi = (self.m.lo, self.m.hi) if lo is None else (lo, hi)
        return mixed_requests(self.rng, self.m.occ, lo, hi, self.m.n_names, n, profile=0 if n == 5000 else None)

    def bounds(self):
        G = self.m.G
        k = self.r(4)
        if k == 0:
            return 0, G
        if k == 1:
            g = self.r(G + 1)
            return g, g                                       # empty
        a, b = sorted((self.r(G + 1), self.r(G + 1)))
        return a, b

    def load_inventory(self):
        G = GS[self.r(len(GS))]
        node_off = unequal_nodes(self.rng, G, max_nodes=6 if self.m.flags & E.FLAG_ALL_NODES else None)
        occ = ((self.rng.next(G) & self.rng.next(G)) & np.uint64(0xFF)).astype(np.uint8)
        self.log.append(f"load_inventory G={G} nodes={len(node_off) - 1}")
        ok, _ = self.attempt("isl_load_inventory", lambda: self.eng.load_inventory(node_off, occ))
        if ok:
            self.m.load_inventory(node_off, occ)

    # -- operations
    def op_batch(self):
        n = self.size()
        req = self.requests(n)
        self.note(f"n={n}")
        ok, got = self.attempt("isl_place_batch", lambda: self.eng.place_batch(req))
        if ok:
            self.check(got, self.m.place_batch(req), "batch")

    def op_range(self):
        lo, hi = self.bounds()
        n = self.size()
        req = self.requests(n, lo, hi)
        self.note(f"[{lo},{hi}) n={n}")
        ok, got = self.attempt("isl_place_batch_range", lambda: self.eng.place_batch_range(lo, hi, req))
        if ok:
            self.check(got, self.m.place_range(lo, hi, req), "range")

    def stream_batches(self):
        batches, total = [], 0
        for _ in range(1 + self.r(3)):
            n = self.size(cap=MAX_BATCH - total)
            batches.append(self.requests(n))
            total += n
        self.note(f"sizes={[len(b) for b in batches]}")
        return batches

    def op_stream(self):
        batches = self.stream_batches()
        ok, got = self.attempt("isl_place_stream", lambda: self.eng.place_stream(batches))
        if ok:
            for b, g in zip(batches, got):
                self.check(g, self.m.place_stream(b), "stream")

    def op_stream_pinned(self):
        batches = self.stream_batches()
        sizes = np.array([len(b) for b in batches], dtype=np.uint32)
        h_in, h_out = E.PinnedArray(int(sizes.sum()), E.REQUEST_DTYPE), E.PinnedArray(int(sizes.sum()), E.RESULT_DTYPE)
        try:
            h_in.array[:] = np.concatenate(batches)
            ok, _ = self.attempt("isl_place_stream", lambda: self.eng.place_stream_ptr(sizes, h_in.ptr, h_out.ptr, device=False))
            if ok:
                self.check(h_out.array.copy(), np.concatenate([self.m.place_stream(b) for b in batches]), "stream pinned")
        finally:
            h_in.free(); h_out.free()

    def device_call(self, batches, symbol, call):
        torch = self.torch
        req = np.concatenate(batches)
        d_in = torch.from_numpy(req.view(np.uint8).copy()).cuda()
        d_out = torch.zeros(len(req) * 8, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        ok, _ = self.attempt(symbol, lambda: call(d_in.data_ptr(), d_out.data_ptr()))
        if ok:
            self.attempt("isl_synchronize", self.eng.synchronize)
            got = d_out.cpu().numpy().view(E.RESULT_DTYPE)
            self.check(got, np.concatenate([self.m.place_stream(b) for b in batches]), symbol)

    def op_stream_device(self):
        batches = self.stream_batches()
        sizes = np.array([len(b) for b in batches], dtype=np.uint32)
        self.device_call(batches, "isl_place_stream_device", lambda i, o: self.eng.place_stream_ptr(sizes, i, o, device=True))

    def op_batch_device(self):
        n = self.size()
        self.note(f"n={n}")
        self.device_call([self.requests(n)], "isl_place_batch_device", lambda i, o: self.eng.place_batch_device(n, i, o))

    def op_gangs(self):
        n = self.size(cap=6000)
        req = self.requests(n)
        cuts = (self.rng.next(max(1, n // 4)) % np.uint64(n)).astype(np.int64)
        off = np.unique(np.r_[0, cuts, n]).astype(np.uint32)
        self.note(f"n={n} gangs={len(off) - 1}")
        ok, got = self.attempt("isl_place_gangs", lambda: self.eng.place_gangs(req, off))
        if ok:
            self.check(got, self.m.place_gangs(req, off), "gangs")

    def op_what_if(self):
        n = self.size()
        plan = self.requests(n)
        self.note(f"n={n}")
        ok, got = self.attempt("isl_what_if", lambda: self.eng.what_if(plan))
        if ok:
            want = self.m.what_if(plan)
            for g, w, what in zip(got, want, ("records", "capacity before", "capacity after")):
                self.check(g, w, ("what_if", what))

    def op_free(self):
        G, k = self.m.G, 1 + self.r(300)
        gpus = np.r_[self.rng.next(k) % np.uint64(G + 3)].astype(np.int64)
        spans = np.zeros(k, dtype=E.SPAN_DTYPE)
        for i, g in enumerate(gpus):
            s, z = (0, 1) if g >= G else mixed_busy(self.m.occ, g)
            if self.r(8) == 0:
                s, z = (5, 4) if self.r(2) else (3, 0)                 # malformed
            spans[i] = (g, s, z, 0)
        self.note(f"spans={k}")
        ok, _ = self.attempt("isl_free_batch", lambda: self.eng.free_batch(spans))
        if ok:
            self.m.free_batch(spans)

    def op_write(self):
        G = self.m.G
        first = self.r(G)
        n = 1 + self.r(min(G - first, 600))
        occ = (self.rng.next(n) & np.uint64(0xFF)).astype(np.uint8)
        self.note(f"[{first},{first + n})")
        ok, _ = self.attempt("isl_write_occupancy", lambda: self.eng.write_occupancy(first, occ))
        if ok:
            self.m.write_occupancy(first, occ)

    def op_capacity(self):
        ok, got = self.attempt("isl_capacity", self.eng.capacity)
        if ok:
            self.check(got, self.m.capacity(), "capacity")

    def op_eval(self):
        profile = self.r(self.m.n_names) | self.r(self.m.n_tables) << 8
        occ = (self.rng.next(300) & np.uint64(0xFF)).astype(np.uint8)
        occ[:2] = (0x80, 0xFF)
        self.note(f"profile={profile:#x}")
        ok, got = self.attempt("isl_eval_starts", lambda: self.eng.eval_starts(profile, occ))
        if ok:
            self.check(got, self.m.eval_starts(profile, occ), "eval_starts")

    def op_snapshot(self):
        if self.attempt("isl_snapshot_occupancy", self.eng.snapshot_occupancy)[0]:
            self.m.snapshot()

    def op_restore(self):
        if self.attempt("isl_restore_occupancy", self.eng.restore_occupancy)[0]:
            self.m.restore()

    def op_partition(self):
        lo, hi = self.bounds()
        self.note(f"[{lo},{hi})")
        if self.attempt("isl_set_partition", lambda: self.eng.set_partition(lo, hi))[0]:
            self.m.set_partition(lo, hi)

    def op_speculation(self):
        mode = self.r(3)
        self.note(f"mode={mode}")
        self.attempt("isl_set_speculation", lambda: self.eng.set_speculation(mode))

    def op_window(self):
        w = self.r(5)
        self.note(f"window={w}")
        self.attempt("isl_set_causal_window", lambda: self.eng.set_causal_window(w))

    def op_set_stream(self):
        s = self.torch.cuda.Stream()
        if self.attempt("isl_set_stream", lambda: self.eng.set_stream(s.cuda_stream))[0]:
            self.op_batch()
            self.attempt("isl_set_stream", lambda: self.eng.set_stream(0))

    def op_node_tables(self):
        n_nodes = len(self.m.node_off) - 1
        nt = (self.rng.next(n_nodes) % np.uint64(self.m.n_tables)).astype(np.uint8)
        if self.attempt("isl_set_node_tables", lambda: self.eng.set_node_tables(nt))[0]:
            self.m.set_node_tables(nt)

    def op_reload(self):
        n_tables = (1, 2, 3)[self.r(3)] if self.n_tables > 1 else 1
        self.note(f"tables={n_tables}")
        load_rows(self.eng, self.m, table_rows(n_tables))

    def op_open(self):
        mb = 1 + self.r(4)
        self.note(f"max_batches={mb}")
        if self.m.lo == self.m.hi:      # open streams on an empty partition are not part of this walk
            self.attempt("isl_set_partition", lambda: self.eng.set_partition(0, self.m.G))
            self.m.set_partition(0, self.m.G)
        if not self.attempt("isl_stream_open", lambda: self.eng.stream_open(mb))[0]:
            return
        self.m.open = [mb, 0, False]
        n_sub = mb if self.r(3) else self.r(mb + 1)            # sometimes closed early
        sizes = [self.size(cap=65536) for _ in range(n_sub)]
        total = max(1, sum(sizes))
        h_in, h_out = E.PinnedArray(total, E.REQUEST_DTYPE), E.PinnedArray(total, E.RESULT_DTYPE)
        refused = sorted(VERIFIED_REFUSED - {"isl_create"})
        try:
            off = 0
            for b, n in enumerate(sizes):
                req = self.requests(n)
                h_in.array[off:off + n] = req
                t = self.eng.stream_submit_ptr(n, h_in.ptr + 8 * off, h_out.ptr + 8 * off)
                self.m.open[1] += 1
                self.m.open[2] = True
                self.probe.ticket = t
                if refused and (b == len(sizes) - 1 or self.r(2)):
                    self.eng.stream_wait(t)
                    # a few refused calls while the stream is open (the sub-state probes passed for every symbol)
                    for name in (refused[self.r(len(refused))] for _ in range(3)):
                        assert self.probe.call(name) == self.m.expected(name), ("during open", name)
                self.eng.stream_wait(t)
                self.check(h_out.array[off:off + n].copy(), self.m.place_stream(req), ("open batch", b))
                off += n
        finally:
            self.eng.stream_close()
            self.m.open = None
        self.note(f"submitted={n_sub}")

    OPS = [("batch", 8), ("range", 3), ("stream", 2), ("stream_pinned", 1), ("stream_device", 1), ("batch_device", 1), ("gangs", 2),
           ("what_if", 2), ("free", 2), ("write", 1), ("capacity", 1), ("eval", 1), ("snapshot", 1), ("restore", 2), ("partition", 2),
           ("speculation", 1), ("window", 1), ("set_stream", 1), ("load_inventory", 1), ("node_tables", 1), ("reload", 1), ("open", 2)]

    def run(self, n_ops):
        names = [name for name, w in self.OPS for _ in range(w)]
        for i in range(n_ops):
            name = names[self.r(len(names))]
            self.log.append(f"{i}: {name}")
            try:
                getattr(self, "load_inventory" if name == "load_inventory" else "op_" + name)()
                if self.m.open is None:
                    self.check_occupancy()
            except AssertionError as err:
                raise AssertionError(f"walk {self.case} seed {self.seed}, operation {i} ({name}): {err}\nlast operations:\n" +
                                     "\n".join(self.log[-20:])) from None

    def close(self):
        self.probe.close()
        self.eng.close()


def mixed_busy(occ, g):
    """The first run of busy slices on GPU g, or slice 0 of an empty GPU."""
    b = int(occ[g])
    if b == 0:
        return 0, 1
    s = (b & -b).bit_length() - 1
    e = s
    while e < 8 and (b >> e) & 1:
        e += 1
    return s, e - s


@pytest.mark.parametrize("case,policy,quirks,n_tables,flags", WALK_CASES)
def test_random_walk(case, policy, quirks, n_tables, flags):
    walk = Walk(case, policy, quirks, n_tables, flags, seed=7000 + WALK_CASES.index((case, policy, quirks, n_tables, flags)))
    try:
        walk.run(N_OPS)
    finally:
        walk.close()
