"""ctypes binding of tests/node_score_fast.cpp, the brute-force restatement of node scoring (ISL_POLICY_MOST_ALLOCATED /
ISL_POLICY_LEAST_ALLOCATED) over nodes and GPUs on flat occupancy bytes.

It is compiled with g++ into a fresh temporary directory once per process (the source tree may be read-only), so it needs no build
step of its own.  ``place`` takes the engine's inputs in canonical order and returns ``(results, occupancy after)``.
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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "node_score_fast.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_node_score_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libnode_score_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p = C.c_void_p
        L.ns_place.restype = C.c_int
        L.ns_place.argtypes = [C.c_uint32, p, C.c_uint32, C.c_uint32, p, p, p, p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                               C.c_uint32, p, p]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def default_sizes(rows2, node_table):
    """Size an unplaced ALLOC reports: that of the first node, in canonical order, whose table has the name."""
    out = np.zeros(rows2.shape[1], dtype=np.uint8)
    for p in range(rows2.shape[1]):
        for t in node_table:
            if rows2[t, p]["n_starts"]:
                out[p] = rows2[t, p]["size"]
                break
    return out


def place(node_off, rows, occ, requests, policy, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0, hi=None):
    """One batch.  ``rows``: [n_profiles] or [n_tables][n_profiles] with ``node_table`` [n_nodes]; [lo, hi): the canonical range."""
    node_off = np.ascontiguousarray(node_off, dtype=np.uint32)
    rows2 = np.ascontiguousarray(np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1]))
    n_nodes = len(node_off) - 1
    node_table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.ascontiguousarray(node_table, dtype=np.uint8)
    dsize = default_sizes(rows2, node_table)
    occ = np.array(occ, dtype=np.uint8, copy=True)
    requests = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    hi = int(node_off[-1]) if hi is None else hi
    rc = lib().ns_place(n_nodes, _ptr(node_off), rows2.shape[0], rows2.shape[1], _ptr(rows2), _ptr(node_table), _ptr(dsize), _ptr(occ),
                        lo, hi, quirks, policy, len(requests), _ptr(requests), _ptr(out))
    assert rc == E.OK
    return out, occ
