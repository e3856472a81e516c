"""ctypes binding of tests/gang_score_all_fast.cpp, the brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_NODE_SCORE |
ISL_FLAG_GANG_NODE_SCORE_ALL engine over flat occupancy bytes: every locality byte 0..255, elastic or not.

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

from gang_locality_oracle import gang_localities
from gang_min_fast import effective_minimum
from preempt_fast import default_sizes

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gang_score_all_fast.cpp")
_lib = None
PER_GANG = None     # `locality` for an ISL_FLAG_GANG_LOCALITY engine: each gang's own byte


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_gang_score_all_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libgang_score_all_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.gsa_place_gangs.restype = C.c_uint64
        L.gsa_place_gangs.argtypes = [u, p, p, u, p, p, p, u, u, u, u, u, p, p, p, p, p]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def place_gangs(node_off, rows, occ, requests, gang_off, policy, locality=PER_GANG, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0,
                hi=None, elastic=False):
    """``locality``: the engine's locality for every gang (``E.GANG_*``: its gang flag, ANY without one), or ``PER_GANG`` for the
    ``start`` byte of each gang's ALLOC members (FLAG_GANG_LOCALITY, L1, B1).  ``elastic``: the engine has FLAG_GANG_MIN_MEMBERS as
    well, and each gang's minimum is the ``size`` byte of its ALLOC members (M1).  ``rows``: [n_profiles] or [n_tables][n_profiles] with
    ``node_table`` [n_nodes]; [lo, hi): the engine's partition (canonical)."""
    node_off = np.ascontiguousarray(node_off, dtype=np.uint32)
    rows2 = np.ascontiguousarray(np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1]))
    n_nodes = len(node_off) - 1
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.ascontiguousarray(node_table, dtype=np.uint8)
    dsize = default_sizes(node_off, rows2, node_table)
    occ = np.array(occ, dtype=np.uint8)
    hi = int(node_off[-1]) if hi is None else hi
    requests = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.ascontiguousarray(gang_off, dtype=np.uint32)
    n_gangs = len(gang_off) - 1
    if locality is PER_GANG:
        loc = np.array([0 if b is None else b for b in gang_localities(requests, gang_off)], dtype=np.uint8)
    else:
        loc = np.full(n_gangs, locality, dtype=np.uint8)
    if elastic:
        mins = effective_minimum(requests, gang_off)
    else:
        mins = np.add.reduceat((requests["op"] == E.OP_ALLOC).astype(np.uint32), gang_off[:-1].astype(np.int64)) if n_gangs else \
            np.zeros(0, dtype=np.uint32)
    mins = np.ascontiguousarray(mins, dtype=np.uint32)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    placed = lib().gsa_place_gangs(n_nodes, _ptr(node_off), _ptr(table), rows2.shape[1], _ptr(rows2), _ptr(dsize), _ptr(occ), lo, hi,
                                   quirks, policy, n_gangs, _ptr(gang_off), _ptr(requests), _ptr(out), _ptr(loc), _ptr(mins))
    return out, occ, int(placed)
