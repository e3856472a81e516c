"""The C-ABI contract of one long-lived engine, as data (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

``CODES``    symbol -> the return code of a well-formed call in each engine state of include/islplace.h: created, profiles only,
             inventory only, ready, and the three sub-states of an open stream — opened and not yet launched; launched with batches
             still due; all max_batches batches submitted and waited (the kernel has left its chunk loop, the stream is not closed).
             An entry is a code, ``VALUE`` for a call that returns a value rather than a code, or a function of a ``Ctx`` where the
             header makes the code depend on the policy, the flags, the partition or the snapshot.
``LEGAL_DURING_OPEN``  the calls an open stream allows; every other call on the engine returns ISL_ESTATE and changes nothing.
``Model``    the state that carries from one call to the next — tables, node map, inventory, partition, snapshot, occupancy — answering
             every placement call through the existing restatements: ``range_oracle.place_range`` / ``RangeFast``,
             ``gang_oracle.fast_place_gangs``, ``oracle.start_for`` and ``range_oracle.capacity_by_hand``.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

import oracle
from instaslice_b200 import engine as E

from gang_oracle import default_sizes, fast_place_gangs
from range_oracle import RangeFast, capacity_by_hand, place_range

STATES = ("created", "profiles", "inventory", "ready")
OPEN_STATES = ("open_unlaunched", "open_partial", "open_drained")
ALL_STATES = STATES + OPEN_STATES
VALUE = "value"

# Calls that stay legal while a stream is open: the stream itself, destroy (closes first) and the pure getters.
LEGAL_DURING_OPEN = frozenset({"isl_stream_submit", "isl_stream_wait", "isl_stream_close", "isl_destroy", "isl_num_gpus", "isl_gpu_to_node",
                               "isl_device_occupancy", "isl_device_results", "isl_abi_version", "isl_strerror", "isl_last_cuda_error",
                               "isl_host_alloc", "isl_host_free"})
# Calls that take no engine: no state can refuse them.
NO_ENGINE = frozenset({"isl_create", "isl_abi_version", "isl_strerror", "isl_host_alloc", "isl_host_free"})


@dataclass(frozen=True)
class Ctx:
    policy: int = E.POLICY_FIRST_FIT
    flags: int = 0
    empty_partition: bool = False
    snapshot: bool = False


def _bestfit(c):
    return c.policy in (E.POLICY_BEST_FIT, E.POLICY_MIN_FRAG)


def _row(created, profiles, inventory, ready, during_open=E.ESTATE):
    return {"created": created, "profiles": profiles, "inventory": inventory, "ready": ready,
            **{s: during_open for s in OPEN_STATES}}


def _always(code):
    return {s: code for s in ALL_STATES}


_ES, _OK = E.ESTATE, E.OK
_IDLE = _row(_OK, _OK, _OK, _OK)                      # legal in every state but an open stream
_INV = _row(_ES, _ES, _OK, _OK)                       # needs an inventory
_READY = _row(_ES, _ES, _ES, _OK)                     # needs profiles and an inventory


def _one_pass_in_partition(state):
    """isl_place_gangs and isl_preempt: a call over the partition, refused on an empty one; a pod on every node (ISL_FLAG_ALL_NODES)
    has no all-or-nothing or eviction meaning."""
    def code(c):
        if c.flags & E.FLAG_ALL_NODES:
            return E.EINVAL                          # checked before the state
        if state != "ready":
            return _ES
        return E.ERANGE if c.empty_partition else _OK
    return code


CODES = {
    "isl_create": _always(_OK),
    "isl_destroy": _always(_OK),
    "isl_set_stream": _IDLE,
    "isl_synchronize": _IDLE,
    "isl_load_profiles": _IDLE,
    "isl_load_profile_tables": _IDLE,
    "isl_set_node_tables": _READY,
    "isl_load_inventory": _IDLE,
    "isl_read_occupancy": _INV,
    "isl_write_occupancy": _INV,
    "isl_snapshot_occupancy": _INV,
    "isl_restore_occupancy": _row(_ES, _ES, lambda c: _OK if c.snapshot else _ES, lambda c: _OK if c.snapshot else _ES),
    "isl_num_gpus": _always(VALUE),
    "isl_gpu_to_node": _always(VALUE),
    "isl_place_batch": _READY,
    "isl_place_batch_device": _READY,
    "isl_place_stream": _READY,
    "isl_place_stream_device": _READY,
    "isl_place_batch_range": _READY,
    "isl_place_gangs": {s: _one_pass_in_partition(s) for s in ALL_STATES},
    "isl_preempt": {s: _one_pass_in_partition(s) for s in ALL_STATES},
    "isl_free_batch": _INV,
    "isl_eval_starts": _row(_ES, _OK, _ES, _OK),
    "isl_set_partition": _INV,
    # the host-carried token of a partitioned batch: first-fit only (best-fit and right-to-left do not partition)
    "isl_place_batch_partitioned": _row(_ES, _ES, _ES, lambda c: E.EINVAL if _bestfit(c) or c.policy == E.POLICY_RIGHT_TO_LEFT else _OK),
    "isl_ipc_inbox_handle": _IDLE,
    "isl_ipc_connect": _IDLE,                        # NULL next handle, no previous rank
    "isl_connect_local": _IDLE,
    "isl_place_stream_partitioned": _row(_ES, _ES, _ES, lambda c: E.EINVAL if _bestfit(c) or c.policy == E.POLICY_RIGHT_TO_LEFT else _OK),
    "isl_device_occupancy": _always(VALUE),
    "isl_get_stats": _IDLE,
    "isl_read_trace": _IDLE,
    "isl_reset_stats": _IDLE,
    "isl_strerror": _always(VALUE),
    "isl_last_cuda_error": _always(VALUE),
    "isl_abi_version": _always(VALUE),
    "isl_stream_open": _row(_ES, _ES, _ES, lambda c: E.EINVAL if _bestfit(c) else _OK),
    "isl_stream_submit": {**_row(_ES, _ES, _ES, _ES), "open_unlaunched": _OK, "open_partial": _OK, "open_drained": E.ERANGE},
    # ticket = the last batch submitted (0 before the first submit)
    "isl_stream_wait": {**_row(_ES, _ES, _ES, _ES), "open_unlaunched": _ES, "open_partial": _OK, "open_drained": _OK},
    "isl_stream_close": {**_row(_ES, _ES, _ES, _ES), "open_unlaunched": _OK, "open_partial": _OK, "open_drained": _OK},
    "isl_set_causal_window": _IDLE,
    "isl_set_speculation": _IDLE,
    "isl_ipc_spec_handle": _IDLE,
    "isl_ipc_connect_spec": _IDLE,                   # world 0: disconnect
    "isl_connect_spec_local": _IDLE,
    "isl_host_alloc": _always(VALUE),
    "isl_host_free": _always(VALUE),
    "isl_device_results": _always(VALUE),
    "isl_ipc_results_handle": _IDLE,
    "isl_ipc_connect_owner": _IDLE,                  # NULL: disconnect
    "isl_connect_owner_local": _IDLE,
    "isl_set_ring_world": _IDLE,
    "isl_capacity": _READY,
    "isl_what_if": _READY,
}


def expected(symbol, state, ctx=Ctx()):
    """The return code (or VALUE) of a well-formed call of ``symbol`` in ``state``."""
    code = CODES[symbol][state]
    return code(ctx) if callable(code) else code


# ---- the state carried from call to call ---------------------------------------------------------------------------------------------
class Model:
    """What one engine holds between calls, in canonical GPU order.  ``rows``: [n] after isl_load_profiles, [n_tables][n] after
    isl_load_profile_tables; ``node_table`` None = every node on table 0; ``lo``/``hi`` the partition; ``snap`` the snapshot or None."""

    def __init__(self, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, flags=0):
        self.policy, self.quirks, self.flags = policy, quirks, flags
        self.rows = None
        self.node_off = None
        self.occ = None
        self.node_table = None
        self.lo = self.hi = 0
        self.snap = None
        self.open = None                 # open stream: [max_batches, submitted, launched]

    # -- state
    @property
    def G(self):
        return 0 if self.node_off is None else int(self.node_off[-1])

    @property
    def n_names(self):
        return self.rows.shape[-1]

    @property
    def n_tables(self):
        return 1 if self.rows.ndim == 1 else self.rows.shape[0]

    def state(self):
        if self.open is not None:
            mb, sub, launched = self.open
            return "open_unlaunched" if not launched else ("open_drained" if sub == mb else "open_partial")
        return ("created", "profiles", "inventory", "ready")[(self.rows is not None) + 2 * (self.node_off is not None)]

    def ctx(self):
        return Ctx(self.policy, self.flags, self.node_off is not None and self.lo == self.hi, self.snap is not None)

    def expected(self, symbol):
        return expected(symbol, self.state(), self.ctx())

    def _table_arg(self):
        """(rows, node_table) as range_oracle takes them."""
        if self.rows.ndim == 1:
            return self.rows, None
        nt = self.node_table if self.node_table is not None else np.zeros(len(self.node_off) - 1, dtype=np.uint8)
        return self.rows, nt

    def gpu_table(self):
        nt = self.node_table if self.node_table is not None else np.zeros(len(self.node_off) - 1, dtype=np.uint8)
        return np.repeat(np.asarray(nt, dtype=np.uint8), np.diff(self.node_off.astype(np.int64)))

    def sizes(self):
        """Size an unplaced ALLOC of each name reports."""
        rows, nt = self._table_arg()
        return default_sizes(rows, nt)

    # -- tables and inventory
    def load_profiles(self, rows):
        self.rows = np.array(rows, dtype=E.PROFILE_DTYPE)
        self.node_table = None                       # every node back on table 0

    def load_inventory(self, node_off, occ):
        self.node_off = np.array(node_off, dtype=np.uint32)
        self.occ = np.array(occ, dtype=np.uint8)
        self.node_table = None
        self.lo, self.hi = 0, self.G
        self.snap = None

    def set_node_tables(self, table_of_node):
        self.node_table = np.array(table_of_node, dtype=np.uint8)

    def set_partition(self, lo, hi):
        self.lo, self.hi = lo, hi

    def write_occupancy(self, first, occ):
        self.occ[first:first + len(occ)] = occ

    def snapshot(self):
        self.snap = self.occ.copy()

    def restore(self):
        self.occ = self.snap.copy()

    # -- placement
    def place_range(self, lo, hi, req, all_nodes=None):
        rows, nt = self._table_arg()
        all_nodes = bool(self.flags & E.FLAG_ALL_NODES) if all_nodes is None else all_nodes
        out, self.occ = place_range(self.node_off, rows, self.occ, lo, hi, req, self.quirks, self.policy, nt, all_nodes=all_nodes)
        return out

    def place_batch(self, req):
        """isl_place_batch inside the partition (ISL_FLAG_ALL_NODES: one pass per node)."""
        return self.place_range(self.lo, self.hi, req)

    def place_stream(self, req):
        """One batch of a stream call, isl_place_batch_device or an open stream: each pod placed once, whatever the flags."""
        return self.place_range(self.lo, self.hi, req, all_nodes=False)

    def place_gangs(self, req, gang_off):
        rows, nt = self._table_arg()
        ref = RangeFast(self.node_off, rows, self.occ, self.lo, self.hi, self.quirks, self.policy, nt)
        out = fast_place_gangs(ref, req, gang_off, self.sizes())
        self.occ = ref.occupancy()
        return out

    def capacity(self):
        return capacity_by_hand(self.rows, self.quirks, self.occ[self.lo:self.hi], None if self.rows.ndim == 1 else self.gpu_table()[self.lo:self.hi])

    def what_if(self, req):
        """(records, capacity before, capacity after); the occupancy is unchanged and the snapshot is gone."""
        live = self.occ.copy()
        before = self.capacity()
        out = self.place_batch(req)
        after = self.capacity()
        self.occ = live
        self.snap = None
        return out, before, after

    def free_batch(self, spans):
        """Spans inside the partition are released; outside or malformed ones change nothing."""
        req = np.zeros(len(spans), dtype=E.REQUEST_DTYPE)
        req["handle"], req["op"], req["start"], req["size"] = spans["gpu"], E.OP_FREE, spans["start"], spans["size"]
        self.place_range(self.lo, self.hi, req, all_nodes=False)

    def eval_starts(self, profile, occ):
        table, p = profile >> 8, profile & 0xFF
        row = self.rows[p] if self.rows.ndim == 1 else self.rows[table, p]
        lut = np.array([oracle.start_for(row, self.quirks, b) for b in range(256)], dtype=np.uint8)
        return lut[np.asarray(occ, dtype=np.uint8)]
