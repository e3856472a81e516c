"""ctypes binding of ``libislplace.so`` (the C ABI declared in ``include/islplace.h``).

This is the same boundary the Go controller binds with cgo (INTEGRATION.md); nothing here computes a
placement.  If the library has not been built (``python -c "import __graft_entry__ as g; g.build()"``)
loading fails loudly — there is no CPU path in the product.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ISL_LIB") or os.path.join(_HERE, "libislplace.so")      # ISL_LIB: A/B builds of the same ABI (tools/)

# ---- constants (mirror include/islplace.h) -------------------------------------------------
ABI_VERSION = 1
MAX_PROFILES = 16
MAX_STARTS = 8
START_NONE = 9
GPU_NONE = 0xFFFFFFFF
PROFILE_UNKNOWN = 0xFF
OK, EINVAL, ENOMEM, ECUDA, ESTATE, ERANGE = 0, -1, -2, -3, -4, -5
POLICY_FIRST_FIT, POLICY_BEST_FIT, POLICY_RIGHT_TO_LEFT, POLICY_MIN_FRAG = 0, 1, 2, 3
POLICY_MOST_ALLOCATED, POLICY_LEAST_ALLOCATED = 4, 5     # node scoring: the kube-scheduler's NodeResourcesFit strategies
NODE_SCORING_MAX_NODES = 1 << 20                         # isl_load_inventory on a node-scoring engine: ERANGE beyond
QUIRK_STRICT_BOUND, QUIRK_POW2_ONLY = 1, 2
QUIRKS_REF_EXACT, QUIRKS_FIXED = 3, 0
OP_ALLOC, OP_FREE, OP_NOOP = 0, 1, 2
ST_PLACED, ST_NO_CAPACITY, ST_BAD_PROFILE, ST_FREED, ST_BAD_SPAN, ST_NOOP, ST_GANG_ABORTED = 0, 1, 2, 3, 4, 5, 6
ST_GANG_TRIMMED = 7     # not placed: its elastic gang committed its leading members without it (include/islplace.h M3)
ST_ALT_SKIPPED = 8      # not tried: an earlier alternative of its pod was placed (FLAG_FIRST_AVAILABLE, include/islplace.h A3)
FLAG_TIMING, FLAG_NO_PIPELINE, FLAG_FORCE_PIPELINE, FLAG_TRACE, FLAG_NO_SMALL, FLAG_ALL_NODES = 1, 2, 4, 8, 16, 32
FLAG_GANG_ONE_NODE = 64     # isl_place_gangs puts every member of a gang on one node (include/islplace.h)
FLAG_GANG_DISTINCT_NODES = 128  # isl_place_gangs puts every member of a gang on a different node (include/islplace.h)
FLAG_GANG_FEW_NODES = 256  # isl_place_gangs puts a gang on one node when one takes it, else on as few nodes as it greedily can
FLAG_GANG_LOCALITY = 512  # isl_place_gangs takes each gang's node locality from its ALLOC members' start byte (GANG_*)
FLAG_GANG_MIN_MEMBERS = 1024  # elastic gangs: a gang commits its leading members once they reach its minimum (the ALLOC size byte)
FLAG_GANG_PREEMPT = 2048  # isl_preempt picks the victims a whole gang (a run of equal handles) needs, or evicts nothing for it
FLAG_GANG_NODE_SCORE = 4096  # on a node-scoring engine isl_place_gangs places gangs by MostAllocated / LeastAllocated (N1-N8)
FLAG_GANG_BALANCED = 8192  # with FLAG_GANG_LOCALITY: a locality of gang_balanced_nodes(k) spreads a gang over the nodes within maxSkew k
FLAG_GANG_NODE_SCORE_ALL = 16384  # with FLAG_GANG_NODE_SCORE: few-node, elastic and balanced gangs are node-scored too (C1-C8)
FLAG_FIRST_AVAILABLE = 32768  # a run of ALLOCs with equal handle is one pod listing alternative profiles; it gets the first that fits (A1-A8)
GANG_ANY_NODES, GANG_ONE_NODE, GANG_FEW_NODES, GANG_DISTINCT_NODES = 0, 1, 2, 3     # node locality of one gang (include/islplace.h L1)
SPEC_AUTO, SPEC_OFF, SPEC_ON = 0, 1, 2

# ---- record layouts -------------------------------------------------------------------------
REQUEST_DTYPE = np.dtype([("handle", "<u4"), ("profile", "u1"), ("op", "u1"), ("start", "u1"), ("size", "u1")])
RESULT_DTYPE = np.dtype([("gpu", "<u4"), ("start", "u1"), ("size", "u1"), ("status", "<u2")])
SPAN_DTYPE = np.dtype([("gpu", "<u4"), ("start", "u1"), ("size", "u1"), ("pad", "<u2")])
PROFILE_DTYPE = np.dtype([("size", "u1"), ("n_starts", "u1"), ("starts", "u1", (8,)), ("pad", "u1", (2,)),
                          ("gi", "<i4"), ("ci", "<i4"), ("cieng", "<i4")])
VICTIM_DTYPE = np.dtype([("gpu", "<u4"), ("start", "u1"), ("size", "u1"), ("priority", "u1"), ("pad", "u1")])
assert REQUEST_DTYPE.itemsize == 8 and RESULT_DTYPE.itemsize == 8 and SPAN_DTYPE.itemsize == 8
assert PROFILE_DTYPE.itemsize == 24 and VICTIM_DTYPE.itemsize == 8


class Config(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("policy", C.c_uint32), ("quirks", C.c_uint32), ("device", C.c_int32),
                ("max_gpus", C.c_uint32), ("max_batch", C.c_uint32), ("flags", C.c_uint32), ("reserved", C.c_uint32)]


class Stats(C.Structure):
    _fields_ = [("batches", C.c_uint64), ("requests", C.c_uint64), ("placed", C.c_uint64), ("no_capacity", C.c_uint64),
                ("freed", C.c_uint64), ("kernel_launches", C.c_uint64), ("chain_steps", C.c_uint64),
                ("chain_gpus_visited", C.c_uint64), ("chain_jumps", C.c_uint64), ("ms_free", C.c_double), ("ms_partition", C.c_double),
                ("ms_sweep", C.c_double), ("ms_commit", C.c_double), ("ms_total", C.c_double), ("scan_placed", C.c_uint64),
                ("spec_chunks", C.c_uint64), ("spec_rounds", C.c_uint64), ("spec_sims", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


# ctypes signature of every symbol include/islplace.h declares; tests check the header against these names and that the library
# exports all of them
_P = C.c_void_p
SIGNATURES = {
    "isl_create": (C.c_int, [C.POINTER(Config), C.POINTER(_P)]),
    "isl_destroy": (C.c_int, [_P]),
    "isl_set_stream": (C.c_int, [_P, _P]),
    "isl_snapshot_occupancy": (C.c_int, [_P]),
    "isl_restore_occupancy": (C.c_int, [_P]),
    "isl_synchronize": (C.c_int, [_P]),
    "isl_load_profiles": (C.c_int, [_P, C.c_uint32, _P]),
    "isl_load_profile_tables": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P]),
    "isl_set_node_tables": (C.c_int, [_P, C.c_uint32, _P]),
    "isl_load_inventory": (C.c_int, [_P, C.c_uint32, _P, _P]),
    "isl_read_occupancy": (C.c_int, [_P, _P]),
    "isl_write_occupancy": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P]),
    "isl_num_gpus": (C.c_uint32, [_P]),
    "isl_gpu_to_node": (C.c_uint32, [_P, C.c_uint32]),
    "isl_place_batch": (C.c_int, [_P, C.c_uint32, _P, _P]),
    "isl_place_batch_device": (C.c_int, [_P, C.c_uint32, _P, _P]),
    "isl_place_stream": (C.c_int, [_P, C.c_uint32, _P, _P, _P]),
    "isl_place_stream_device": (C.c_int, [_P, C.c_uint32, _P, _P, _P]),
    "isl_free_batch": (C.c_int, [_P, C.c_uint32, _P]),
    "isl_eval_starts": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P, _P]),
    "isl_set_partition": (C.c_int, [_P, C.c_uint32, C.c_uint32]),
    "isl_place_batch_partitioned": (C.c_int, [_P, C.c_uint32, _P, _P, _P, _P]),
    "isl_ipc_inbox_handle": (C.c_int, [_P, _P]),
    "isl_ipc_connect": (C.c_int, [_P, _P, C.c_int]),
    "isl_connect_local": (C.c_int, [_P, _P, C.c_int]),
    "isl_place_stream_partitioned": (C.c_int, [_P, C.c_uint32, _P, _P, _P, C.c_uint32]),
    "isl_device_occupancy": (_P, [_P]),
    "isl_get_stats": (C.c_int, [_P, C.POINTER(Stats)]),
    "isl_read_trace": (C.c_int, [_P, _P, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]),
    "isl_reset_stats": (C.c_int, [_P]),
    "isl_strerror": (C.c_char_p, [C.c_int]),
    "isl_last_cuda_error": (C.c_char_p, [_P]),
    "isl_abi_version": (C.c_uint32, []),
    "isl_place_batch_range": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_uint32, _P, _P]),
    "isl_place_gangs": (C.c_int, [_P, C.c_uint32, _P, _P, _P]),
    "isl_preempt": (C.c_int, [_P, C.c_uint32, _P, _P, C.c_uint32, _P, _P, _P]),
    "isl_stream_open": (C.c_int, [_P, C.c_uint32]),
    "isl_stream_submit": (C.c_int, [_P, C.c_uint32, _P, _P, C.POINTER(C.c_uint32)]),
    "isl_stream_wait": (C.c_int, [_P, C.c_uint32]),
    "isl_stream_close": (C.c_int, [_P]),
    "isl_set_causal_window": (C.c_int, [_P, C.c_uint32]),
    "isl_set_speculation": (C.c_int, [_P, C.c_uint32]),
    "isl_ipc_spec_handle": (C.c_int, [_P, C.c_void_p]),
    "isl_ipc_connect_spec": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]),
    "isl_connect_spec_local": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]),
    "isl_host_alloc": (_P, [C.c_size_t]),
    "isl_host_free": (None, [_P]),
    "isl_device_results": (_P, [_P]),
    "isl_ipc_results_handle": (C.c_int, [_P, _P]),
    "isl_ipc_connect_owner": (C.c_int, [_P, _P]),
    "isl_connect_owner_local": (C.c_int, [_P, _P]),
    "isl_set_ring_world": (C.c_int, [_P, C.c_uint32]),
    "isl_capacity": (C.c_int, [_P, _P]),
    "isl_what_if": (C.c_int, [_P, C.c_uint32, _P, _P, _P, _P]),
}

_lib = None


def load_library(path: str = LIB_PATH):
    """dlopen the engine.  Raises (never falls back) when the CUDA library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise ImportError(f"{path} not built: run __graft_entry__.build() (nvcc, sm_90a). There is no CPU fallback.")
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            if os.environ.get("ISL_LIB"):       # an A/B build of an older revision (tools/): entry points added since are simply absent
                continue
            raise
        fn.restype, fn.argtypes = res, args
    _lib = lib
    return lib


class EngineError(RuntimeError):
    def __init__(self, code, what, detail=""):
        super().__init__(f"{what}: {load_library().isl_strerror(code).decode()} ({code}) {detail}".strip())
        self.code = code


def gang_balanced_nodes(max_skew: int) -> int:
    """The locality byte of a balanced gang with maxSkew ``max_skew`` (1..252) on a ``FLAG_GANG_BALANCED`` engine
    (ISL_GANG_BALANCED_NODES, include/islplace.h B1): ``topologySpreadConstraints.maxSkew`` on ``kubernetes.io/hostname``."""
    if isinstance(max_skew, bool) or int(max_skew) != max_skew or not 1 <= max_skew <= 252:
        raise ValueError("maxSkew is 1..252")
    return 3 + int(max_skew)


def make_profiles(table, right_to_left: bool = False) -> np.ndarray:
    """``tables.A100_40GB``-style rows -> isl_profile records (duplicate starts dropped, order kept).

    ``right_to_left``: the start search takes the first legal start in ROW order (:343-383), so a right-to-left placement inside a
    GPU (the policy the reference only stubs, :464-469) is the same engine fed with the rows reversed — SURVEY 8f-4."""
    rows = np.zeros(len(table), dtype=PROFILE_DTYPE)
    for i, (_name, size, starts, gi) in enumerate(table):
        uniq = []
        for s in (list(starts)[::-1] if right_to_left else starts):
            if s not in uniq:
                uniq.append(s)
        rows[i]["size"] = size
        rows[i]["n_starts"] = len(uniq)
        rows[i]["starts"][: len(uniq)] = uniq
        rows[i]["gi"], rows[i]["ci"], rows[i]["cieng"] = gi, gi, 0
    return rows


def make_profile_tables(table_list):
    """Several per-node tables (heterogeneous cluster) -> (profile names, isl_profile records [n_tables][n_names]).

    The name list is the union of the tables' profile names in order of first appearance; a table that has no row
    of a name gets ``n_starts == 0`` there (the reference finds no Migplacement row on such a node and returns 9)."""
    names = []
    for table in table_list:
        for name, *_ in table:
            if name not in names:
                names.append(name)
    rows = np.zeros((len(table_list), len(names)), dtype=PROFILE_DTYPE)
    for t, table in enumerate(table_list):
        seen = set()
        for row in table:
            if row[0] in seen:            # the start search uses the FIRST row with a name (:332-340)
                continue
            seen.add(row[0])
            rows[t, names.index(row[0])] = make_profiles([row])[0]
    return names, rows


class PinnedArray:
    """A numpy view of mapped pinned host memory from the engine's own allocator (isl_host_alloc) — what the Go shim uses for the
    buffers of an open stream."""

    def __init__(self, n: int, dtype):
        lib = load_library()
        self.dtype = np.dtype(dtype)
        self.nbytes = max(1, n) * self.dtype.itemsize
        self.ptr = lib.isl_host_alloc(self.nbytes)
        if not self.ptr:
            raise MemoryError("isl_host_alloc failed")
        self.array = np.frombuffer((C.c_uint8 * self.nbytes).from_address(self.ptr), dtype=self.dtype, count=n)

    def free(self):
        if getattr(self, "ptr", None):
            self.array = None
            load_library().isl_host_free(C.c_void_p(self.ptr))
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class Engine:
    """One placement engine on one H100 (thin, 1:1 over the C ABI)."""

    def __init__(self, max_gpus: int, max_batch: int, policy: int = POLICY_FIRST_FIT, quirks: int = QUIRKS_REF_EXACT,
                 device: int = -1, timing: bool = False, flags: int = 0):
        self._lib = load_library()
        cfg = Config(ABI_VERSION, policy, quirks, device, max_gpus, max_batch, (FLAG_TIMING if timing else 0) | flags, 0)
        h = C.c_void_p()
        rc = self._lib.isl_create(C.byref(cfg), C.byref(h))
        if rc != OK:
            raise EngineError(rc, "isl_create")
        self._h = h
        self.max_batch = max_batch
        self.flags = cfg.flags

    # -- lifetime
    def close(self):
        if getattr(self, "_h", None):
            self._lib.isl_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != OK:
            detail = self._lib.isl_last_cuda_error(self._h).decode() if rc == ECUDA else ""
            raise EngineError(rc, what, detail)

    def set_stream(self, cuda_stream: int):
        self._check(self._lib.isl_set_stream(self._h, C.c_void_p(cuda_stream)), "isl_set_stream")

    def synchronize(self):
        self._check(self._lib.isl_synchronize(self._h), "isl_synchronize")

    # -- tables / inventory
    def load_profiles(self, rows: np.ndarray):
        rows = np.ascontiguousarray(rows, dtype=PROFILE_DTYPE)
        self._check(self._lib.isl_load_profiles(self._h, len(rows), _ptr(rows)), "isl_load_profiles")

    def load_profile_tables(self, rows2d: np.ndarray):
        """[n_tables][n_profile_names] rows of a heterogeneous cluster (``make_profile_tables``)."""
        rows2d = np.ascontiguousarray(rows2d, dtype=PROFILE_DTYPE)
        self._check(self._lib.isl_load_profile_tables(self._h, rows2d.shape[0], rows2d.shape[1], _ptr(rows2d)), "isl_load_profile_tables")

    def set_node_tables(self, node_table):
        node_table = np.ascontiguousarray(node_table, dtype=np.uint8)
        self._check(self._lib.isl_set_node_tables(self._h, len(node_table), _ptr(node_table)), "isl_set_node_tables")

    def load_inventory(self, node_off, occ):
        """Raises ``EngineError`` with code ``ERANGE`` for more GPUs than ``max_gpus``, and on a node-scoring engine for more than
        ``NODE_SCORING_MAX_NODES`` nodes (empty ones count); the engine then keeps its previous inventory."""
        node_off =np.ascontiguousarray(node_off, dtype=np.uint32)
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        assert len(occ) == int(node_off[-1])
        self._check(self._lib.isl_load_inventory(self._h, len(node_off) - 1, _ptr(node_off), _ptr(occ)), "isl_load_inventory")

    def read_occupancy(self) -> np.ndarray:
        out = np.empty(self.num_gpus, dtype=np.uint8)
        self._check(self._lib.isl_read_occupancy(self._h, _ptr(out)), "isl_read_occupancy")
        return out

    def write_occupancy(self, first_gpu: int, occ):
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        self._check(self._lib.isl_write_occupancy(self._h, first_gpu, len(occ), _ptr(occ)), "isl_write_occupancy")

    @property
    def num_gpus(self) -> int:
        return int(self._lib.isl_num_gpus(self._h))

    def gpu_to_node(self, gpu: int) -> int:
        return int(self._lib.isl_gpu_to_node(self._h, gpu))

    # -- hot path
    def place_batch(self, requests: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """Host buffers in, host buffers out (the call the Go shim makes).  On an engine created with ``FLAG_FIRST_AVAILABLE`` a run of
        consecutive ALLOCs with equal ``handle`` is one pod whose profiles are alternatives in order of preference: the first that fits
        is PLACED, the ones before it keep their unplaced records and the ones after it report ``ST_ALT_SKIPPED`` (include/islplace.h
        A1-A8)."""
        requests = np.ascontiguousarray(requests, dtype=REQUEST_DTYPE)
        if out is None:
            out = np.empty(len(requests), dtype=RESULT_DTYPE)
        self._check(self._lib.isl_place_batch(self._h, len(requests), _ptr(requests), _ptr(out)), "isl_place_batch")
        return out

    def place_stream(self, batches: list) -> list:
        """A stream of batches in one call (host buffers); same results as place_batch per batch, pipelined on the device.
        (numpy arrays are pageable: the H2D / D2H overlap of isl_place_stream needs pinned buffers, see place_stream_ptr.)"""
        sizes = np.array([len(b) for b in batches], dtype=np.uint32)
        req = np.ascontiguousarray(np.concatenate(batches) if len(batches) else np.zeros(0, dtype=REQUEST_DTYPE), dtype=REQUEST_DTYPE)
        out = np.empty(len(req), dtype=RESULT_DTYPE)
        self._check(self._lib.isl_place_stream(self._h, len(sizes), _ptr(sizes), _ptr(req), _ptr(out)), "isl_place_stream")
        return np.split(out, np.cumsum(sizes)[:-1]) if len(sizes) else []

    def place_stream_ptr(self, sizes: np.ndarray, in_ptr: int, out_ptr: int, device: bool):
        sizes = np.ascontiguousarray(sizes, dtype=np.uint32)
        fn = self._lib.isl_place_stream_device if device else self._lib.isl_place_stream
        self._check(fn(self._h, len(sizes), _ptr(sizes), C.c_void_p(in_ptr), C.c_void_p(out_ptr)), "isl_place_stream")

    def place_batch_ptr(self, n: int, in_ptr: int, out_ptr: int):
        """Host buffers by raw address (pinned torch tensors in the bench)."""
        self._check(self._lib.isl_place_batch(self._h, n, C.c_void_p(in_ptr), C.c_void_p(out_ptr)), "isl_place_batch")

    def place_batch_device(self, n: int, d_in: int, d_out: int):
        self._check(self._lib.isl_place_batch_device(self._h, n, C.c_void_p(d_in), C.c_void_p(d_out)), "isl_place_batch_device")

    def place_batch_range(self, lo: int, hi: int, requests: np.ndarray, out: np.ndarray | None = None) -> np.ndarray:
        """place_batch restricted to the canonical GPU range [lo, hi) (one node's GPUs) under one engine lock."""
        requests = np.ascontiguousarray(requests, dtype=REQUEST_DTYPE)
        if out is None:
            out = np.empty(len(requests), dtype=RESULT_DTYPE)
        self._check(self._lib.isl_place_batch_range(self._h, lo, hi, len(requests), _ptr(requests), _ptr(out)), "isl_place_batch_range")
        return out

    def place_gangs(self, requests: np.ndarray, gang_off, locality=None, min_members=None) -> np.ndarray:
        """All-or-nothing groups: gang i is ``requests[gang_off[i]:gang_off[i + 1]]`` (``gang_off[0] == 0``, no empty gang, the last
        offset is ``len(requests)``).  A gang commits only when every ALLOC member is placed; otherwise the first member that did not fit
        keeps its record and every other ALLOC member reports ``ST_GANG_ABORTED`` (include/islplace.h).  On an engine created with
        ``FLAG_GANG_ONE_NODE`` every gang lands on one node, the first in scan order that takes it whole, and the member at the depth no
        node gets past keeps its record.  On an engine created with ``FLAG_GANG_DISTINCT_NODES`` every member of a gang lands on a
        different node, resolved greedily member by member, and the first member with no GPU on an unused node keeps its record.  On an
        engine created with ``FLAG_GANG_FEW_NODES`` a gang goes to one node when one takes it whole, else in rounds: each round the node
        that places the most of the remaining members takes them; when no node places the next member, that member keeps its record.

        On an engine created with ``FLAG_GANG_LOCALITY`` each gang is placed by its own locality, the ``start`` byte of its ALLOC members
        (``GANG_ANY_NODES``, ``GANG_ONE_NODE``, ``GANG_FEW_NODES`` or ``GANG_DISTINCT_NODES``).  ``locality``: one such value per gang,
        written into the ``start`` of the ALLOC members of a copy of ``requests``; it needs an engine created with the flag.

        On an engine created with ``FLAG_GANG_MIN_MEMBERS`` a gang may commit its leading members: when its locality's rules stop at
        ALLOC member f and f reaches the gang's minimum m' (the ``size`` byte m of its ALLOC members; m' = m for 0 < m < k, else every
        one of its k members), the first f members are placed, member f keeps its record and the members after it report
        ``ST_GANG_TRIMMED`` (include/islplace.h M1-M7).  ``min_members``: one m in 0..255 per gang, written into the ``size`` of the
        ALLOC members of a copy of ``requests``; it needs an engine created with the flag.

        On a ``POLICY_MOST_ALLOCATED`` or ``POLICY_LEAST_ALLOCATED`` engine created with ``FLAG_GANG_NODE_SCORE`` the gangs are placed by
        the node score (include/islplace.h N1-N8): any-node and distinct-node members one by one, each on the best-scored node that admits
        it (ties to the lowest node) and there on its first admitting GPU; a one-node gang on the node that takes it whole with the best
        score for the gang's slices taken as one pod.  Its locality is ``FLAG_GANG_ONE_NODE``, ``FLAG_GANG_DISTINCT_NODES``, each gang's
        own under ``FLAG_GANG_LOCALITY`` (``GANG_FEW_NODES`` is refused), or any node.

        With ``FLAG_GANG_NODE_SCORE_ALL`` as well such an engine places every gang kind (include/islplace.h C1-C8): ``FLAG_GANG_FEW_NODES``
        or ``GANG_FEW_NODES``, ``FLAG_GANG_MIN_MEMBERS`` and ``FLAG_GANG_BALANCED``.  Each kind keeps its own first criterion (a few-node
        round's depth, an elastic trim's depth, a balanced member's nodes within the skew); the node score breaks the ties below it, where
        a first-fit engine takes scan order, and the lowest node breaks the ties of the score.

        On an engine created with ``FLAG_GANG_LOCALITY | FLAG_GANG_BALANCED`` a locality of ``gang_balanced_nodes(k)`` (4..255) spreads
        the gang's members over the nodes: each member goes, by the engine's policy, to a node whose count of the gang's earlier members
        is at most the least such count over the nodes that admit it plus k - 1 (include/islplace.h B1-B8)."""
        requests = np.ascontiguousarray(requests, dtype=REQUEST_DTYPE)
        gang_off = np.ascontiguousarray(gang_off, dtype=np.uint32)
        if len(gang_off) == 0 or int(gang_off[-1]) != len(requests):
            raise ValueError("gang_off must have n_gangs + 1 entries ending at len(requests)")
        if locality is not None:
            if not self.flags & FLAG_GANG_LOCALITY:
                raise ValueError("a locality per gang needs an engine created with FLAG_GANG_LOCALITY")
            locality = np.asarray(locality, dtype=np.int64)
            if len(locality) != len(gang_off) - 1:
                raise ValueError("one locality per gang")
            if self.flags & FLAG_GANG_NODE_SCORE and not self.flags & FLAG_GANG_NODE_SCORE_ALL and (locality == GANG_FEW_NODES).any():
                raise ValueError("few-node gangs are not node-scored (FLAG_GANG_NODE_SCORE)")
            if self.flags & FLAG_GANG_BALANCED and len(locality) and (locality.min() < 0 or locality.max() > 255):
                raise ValueError("a locality is 0..255 (gang_balanced_nodes(1..252) above GANG_DISTINCT_NODES)")
            requests = requests.copy()
            per_request = np.repeat(locality, np.diff(gang_off.astype(np.int64)))
            alloc = requests["op"] == OP_ALLOC
            requests["start"][alloc] = per_request[alloc].astype(np.uint8)
        if min_members is not None:
            if not self.flags & FLAG_GANG_MIN_MEMBERS:
                raise ValueError("a minimum per gang needs an engine created with FLAG_GANG_MIN_MEMBERS")
            min_members = np.asarray(min_members, dtype=np.int64).reshape(-1)
            if len(min_members) != len(gang_off) - 1:
                raise ValueError("one minimum per gang")
            if len(min_members) and (min_members.min() < 0 or min_members.max() > 255):
                raise ValueError("a gang's minimum is 0..255")
            requests = requests.copy()
            per_request = np.repeat(min_members, np.diff(gang_off.astype(np.int64)))
            alloc = requests["op"] == OP_ALLOC
            requests["size"][alloc] = per_request[alloc].astype(np.uint8)
        out = np.empty(len(requests), dtype=RESULT_DTYPE)
        self._check(self._lib.isl_place_gangs(self._h, len(gang_off) - 1, _ptr(gang_off), _ptr(requests), _ptr(out)), "isl_place_gangs")
        return out

    def preempt(self, requests: np.ndarray, priority, victims: np.ndarray, gang_off=None, locality=None):
        """Priority preemption query (isl_preempt): for each ALLOC in ``requests`` at ``priority[i]`` (uint8, higher = more important),
        the GPU and start it would take once the lower-priority ``victims`` (VICTIM_DTYPE) listed in ``evict[i]`` are gone.  Returns
        ``(results, evict)``, ``evict`` an [n, 8] uint32 array of victim indices padded with GPU_NONE.  Changes no engine state.

        On an engine created with ``FLAG_GANG_PREEMPT`` the runs of equal ``handle`` are gangs: a gang gets victims for every ALLOC
        member or for none (include/islplace.h P1-P8), its members share one priority, and a one-node gang goes to the node whose
        victims cost least.  ``gang_off``: gang i is ``requests[gang_off[i]:gang_off[i + 1]]``, written as gang indices into the
        ``handle`` of a copy; ``locality``: one ``GANG_*`` value per gang (0, 1 or 3), written into the ``start`` of the ALLOC members of
        the copy, which needs an engine created with ``FLAG_GANG_LOCALITY`` as well.  Both need an engine created with the flag."""
        requests = np.ascontiguousarray(requests, dtype=REQUEST_DTYPE)
        priority = np.ascontiguousarray(priority, dtype=np.uint8)
        victims = np.ascontiguousarray(victims, dtype=VICTIM_DTYPE)
        if len(priority) != len(requests):
            raise ValueError("one priority per request")
        if gang_off is not None or locality is not None:
            if not self.flags & FLAG_GANG_PREEMPT:
                raise ValueError("gangs in isl_preempt need an engine created with FLAG_GANG_PREEMPT")
            requests = requests.copy()
        if gang_off is not None:
            gang_off = np.asarray(gang_off, dtype=np.int64)
            if len(gang_off) == 0 or gang_off[0] != 0 or int(gang_off[-1]) != len(requests) or (np.diff(gang_off) <= 0).any():
                raise ValueError("gang_off must start at 0, rise strictly and end at len(requests)")
            requests["handle"] = np.repeat(np.arange(len(gang_off) - 1), np.diff(gang_off)).astype(np.uint32)
        if locality is not None:
            if not self.flags & FLAG_GANG_LOCALITY:
                raise ValueError("a locality per gang needs an engine created with FLAG_GANG_LOCALITY")
            if gang_off is None:
                raise ValueError("a locality per gang needs gang_off")
            locality = np.asarray(locality, dtype=np.int64)
            if len(locality) != len(gang_off) - 1:
                raise ValueError("one locality per gang")
            per_request = np.repeat(locality, np.diff(gang_off))
            alloc = requests["op"] == OP_ALLOC
            requests["start"][alloc] = per_request[alloc].astype(np.uint8)
        out = np.empty(len(requests), dtype=RESULT_DTYPE)
        evict = np.empty((len(requests), 8), dtype=np.uint32)
        self._check(self._lib.isl_preempt(self._h, len(requests), _ptr(requests), _ptr(priority), len(victims), _ptr(victims), _ptr(out),
                                          _ptr(evict)), "isl_preempt")
        return out, evict

    # -- open streams (the causal feed)
    def stream_open(self, max_batches: int):
        self._check(self._lib.isl_stream_open(self._h, max_batches), "isl_stream_open")

    def stream_submit_ptr(self, n: int, in_ptr: int, out_ptr: int) -> int:
        t = C.c_uint32()
        self._check(self._lib.isl_stream_submit(self._h, n, C.c_void_p(in_ptr), C.c_void_p(out_ptr), C.byref(t)), "isl_stream_submit")
        return t.value

    def stream_wait(self, ticket: int):
        self._check(self._lib.isl_stream_wait(self._h, ticket), "isl_stream_wait")

    def stream_close(self):
        self._check(self._lib.isl_stream_close(self._h), "isl_stream_close")

    def set_causal_window(self, window: int):
        self._check(self._lib.isl_set_causal_window(self._h, window), "isl_set_causal_window")

    def ipc_spec_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._check(self._lib.isl_ipc_spec_handle(self._h, buf), "isl_ipc_spec_handle")
        return buf.raw

    def ipc_connect_spec(self, world: int, rank: int, handles: list, bounds):
        """``handles``: the 64-byte ``ipc_spec_handle()`` of every rank; ``bounds``: world + 1 canonical GPU indices."""
        blob = C.create_string_buffer(b"".join(h if h else b"\0" * 64 for h in handles), 64 * world)
        b = np.ascontiguousarray(bounds, dtype=np.uint32)
        self._check(self._lib.isl_ipc_connect_spec(self._h, world, rank, blob, _ptr(b)), "isl_ipc_connect_spec")

    def connect_spec_local(self, world: int, rank: int, engines: list, bounds):
        arr = (C.c_void_p * world)(*[e._h for e in engines])
        b = np.ascontiguousarray(bounds, dtype=np.uint32)
        self._check(self._lib.isl_connect_spec_local(self._h, world, rank, arr, _ptr(b)), "isl_connect_spec_local")

    def set_speculation(self, mode: int):
        """SPEC_AUTO / SPEC_OFF / SPEC_ON: speculative rounds inside the segment pipeline (include/islplace.h)."""
        self._check(self._lib.isl_set_speculation(self._h, mode), "isl_set_speculation")

    def free_batch(self, spans: np.ndarray):
        spans = np.ascontiguousarray(spans, dtype=SPAN_DTYPE)
        self._check(self._lib.isl_free_batch(self._h, len(spans), _ptr(spans)), "isl_free_batch")

    def eval_starts(self, profile: int, occ: np.ndarray) -> np.ndarray:
        occ = np.ascontiguousarray(occ, dtype=np.uint8)
        out = np.empty(len(occ), dtype=np.uint8)
        self._check(self._lib.isl_eval_starts(self._h, profile, len(occ), _ptr(occ), _ptr(out)), "isl_eval_starts")
        return out

    # -- partitioned inventory
    def set_partition(self, lo: int, hi: int):
        self._check(self._lib.isl_set_partition(self._h, lo, hi), "isl_set_partition")

    def place_batch_partitioned(self, n: int, d_in: int, d_out: int, d_heads_in: int | None, d_heads_out: int):
        self._check(self._lib.isl_place_batch_partitioned(self._h, n, C.c_void_p(d_in), C.c_void_p(d_out),
                                                          C.c_void_p(d_heads_in or 0), C.c_void_p(d_heads_out)),
                    "isl_place_batch_partitioned")

    def ipc_inbox_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._check(self._lib.isl_ipc_inbox_handle(self._h, buf), "isl_ipc_inbox_handle")
        return buf.raw

    def ipc_connect(self, next_handle: bytes | None, has_prev: bool):
        self._check(self._lib.isl_ipc_connect(self._h, next_handle, 1 if has_prev else 0), "isl_ipc_connect")

    def connect_local(self, nxt: "Engine | None", has_prev: bool):
        self._check(self._lib.isl_connect_local(self._h, nxt._h if nxt is not None else None, 1 if has_prev else 0), "isl_connect_local")

    def place_stream_partitioned(self, sizes: np.ndarray, d_in: int, d_out: int, stream_id: int):
        sizes = np.ascontiguousarray(sizes, dtype=np.uint32)
        self._check(self._lib.isl_place_stream_partitioned(self._h, len(sizes), _ptr(sizes), C.c_void_p(d_in), C.c_void_p(d_out), stream_id),
                    "isl_place_stream_partitioned")

    def device_results(self) -> int:
        return int(self._lib.isl_device_results(self._h) or 0)

    def ipc_results_handle(self) -> bytes:
        buf = C.create_string_buffer(64)
        self._check(self._lib.isl_ipc_results_handle(self._h, buf), "isl_ipc_results_handle")
        return buf.raw

    def ipc_connect_owner(self, handle: bytes | None):
        self._check(self._lib.isl_ipc_connect_owner(self._h, handle), "isl_ipc_connect_owner")

    def connect_owner_local(self, owner: "Engine | None"):
        self._check(self._lib.isl_connect_owner_local(self._h, owner._h if owner is not None else None), "isl_connect_owner_local")

    def set_ring_world(self, world: int):
        self._check(self._lib.isl_set_ring_world(self._h, world), "isl_set_ring_world")

    def device_occupancy(self) -> int:
        return int(self._lib.isl_device_occupancy(self._h) or 0)

    def snapshot_occupancy(self):
        """What-if queries: keep a device-side copy of the occupancy ... (see restore_occupancy)."""
        self._check(self._lib.isl_snapshot_occupancy(self._h), "isl_snapshot_occupancy")

    def capacity(self) -> np.ndarray:
        """Per profile: how many more pods of that profile alone the inventory could still take."""
        cap = np.zeros(MAX_PROFILES, dtype=np.uint64)
        self._check(self._lib.isl_capacity(self._h, _ptr(cap)), "isl_capacity")
        return cap

    def what_if(self, plan: np.ndarray):
        """Resolve ``plan`` against the live occupancy, then put the live state back.  Returns (results, capacity before, capacity after)."""
        plan = np.ascontiguousarray(plan, dtype=REQUEST_DTYPE)
        out = np.empty(len(plan), dtype=RESULT_DTYPE)
        before, after = np.zeros(MAX_PROFILES, dtype=np.uint64), np.zeros(MAX_PROFILES, dtype=np.uint64)
        self._check(self._lib.isl_what_if(self._h, len(plan), _ptr(plan), _ptr(out), _ptr(before), _ptr(after)), "isl_what_if")
        return out, before, after

    def restore_occupancy(self):
        """... and put it back after any number of placement calls (defragmentation planning, SURVEY 8f-4)."""
        self._check(self._lib.isl_restore_occupancy(self._h), "isl_restore_occupancy")

    # -- diagnostics
    def read_trace(self) -> np.ndarray:
        """[chunk][segment][12] of the last stream call (FLAG_TRACE): globaltimer ns of sweep done, token in, token out, commit done,
        chain start, chain end; the decisions of the cell; jumps | visited << 32; ns of heads done, windows staged; 2 spare."""
        nc, ns = C.c_uint32(), C.c_uint32()
        self._check(self._lib.isl_read_trace(self._h, None, 0, C.byref(nc), C.byref(ns)), "isl_read_trace")
        out = np.zeros((nc.value, ns.value, 12), dtype=np.uint64)
        if out.size:
            self._check(self._lib.isl_read_trace(self._h, _ptr(out), out.size, C.byref(nc), C.byref(ns)), "isl_read_trace")
        return out

    def stats(self) -> dict:
        s = Stats()
        self._check(self._lib.isl_get_stats(self._h, C.byref(s)), "isl_get_stats")
        return s.as_dict()

    def reset_stats(self):
        self._check(self._lib.isl_reset_stats(self._h), "isl_reset_stats")
