"""ctypes binding of tests/gang_score_fast.cpp, the brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE engine over
flat occupancy bytes.

It is compiled with g++ into a fresh temporary directory once per process (the source tree may be read-only), so it needs no build step
of its own.  ``place_gangs`` takes the engine's inputs in canonical order and returns ``(records, occupancy after, members placed)``.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from instaslice_b200 import engine as E

from preempt_fast import default_sizes

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gang_score_fast.cpp")
_lib = None
PER_GANG = 4        # `locality` for an ISL_FLAG_GANG_LOCALITY engine: each gang's own byte


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_gang_score_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libgang_score_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.gsf_place_gangs.restype = C.c_uint64
        L.gsf_place_gangs.argtypes = [u, p, p, u, p, p, p, u, u, u, u, u, u, p, p, p]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def locality_of(flags):
    """The ``locality`` argument of an engine created with ``flags``."""
    if flags & E.FLAG_GANG_LOCALITY:
        return PER_GANG
    if flags & E.FLAG_GANG_ONE_NODE:
        return E.GANG_ONE_NODE
    if flags & E.FLAG_GANG_DISTINCT_NODES:
        return E.GANG_DISTINCT_NODES
    return E.GANG_ANY_NODES


def place_gangs(node_off, rows, occ, requests, gang_off, policy, locality, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0, hi=None):
    """``rows``: [n_profiles] or [n_tables][n_profiles] with ``node_table`` [n_nodes]; [lo, hi): the engine's partition (canonical);
    ``locality``: GANG_ANY_NODES, GANG_ONE_NODE or GANG_DISTINCT_NODES for every gang, or PER_GANG for each gang's ``start`` byte."""
    node_off = np.ascontiguousarray(node_off, dtype=np.uint32)
    rows2 = np.ascontiguousarray(np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1]))
    n_nodes = len(node_off) - 1
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.ascontiguousarray(node_table, dtype=np.uint8)
    dsize = default_sizes(node_off, rows2, node_table)
    occ = np.array(occ, dtype=np.uint8)
    hi = int(node_off[-1]) if hi is None else hi
    requests = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.ascontiguousarray(gang_off, dtype=np.uint32)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    placed = lib().gsf_place_gangs(n_nodes, _ptr(node_off), _ptr(table), rows2.shape[1], _ptr(rows2), _ptr(dsize), _ptr(occ), lo, hi, quirks,
                                   policy, locality, len(gang_off) - 1, _ptr(gang_off), _ptr(requests), _ptr(out))
    return out, occ, int(placed)
