"""ctypes binding of tests/gang_few_fast.cpp, the brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_FEW_NODES engine over
flat occupancy bytes.

It is compiled with g++ into a fresh temporary directory once per process (the source tree may be read-only), so it needs no build step
of its own.  ``place_gangs`` takes the engine's inputs in canonical order and returns ``(records, occupancy after)``; with
``rounds=True`` also, per request, the round that placed it in a committed gang (-1 for none).
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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gang_few_fast.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_gang_few_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libgang_few_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.gff_place_gangs.restype = None
        L.gff_place_gangs.argtypes = [u, p, p, u, p, p, p, u, u, u, u, u, p, p, p, u, p]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def place_gangs(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
                lo=0, hi=None, memo=True, rounds=False):
    """``rows``: [n_profiles] or [n_tables][n_profiles] with ``node_table`` [n_nodes]; [lo, hi): the engine's partition (canonical);
    ``memo``: ISL_POLICY_MIN_FRAG scores are walked once per (table, profile, byte) and remembered, which 2^20-GPU calls need."""
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
    rnd = np.zeros(len(requests), dtype=np.int32)
    lib().gff_place_gangs(n_nodes, _ptr(node_off), _ptr(table), rows2.shape[1], _ptr(rows2), _ptr(dsize), _ptr(occ), lo, hi, quirks, policy,
                          len(gang_off) - 1, _ptr(gang_off), _ptr(requests), _ptr(out), int(memo), _ptr(rnd))
    return (out, occ, rnd) if rounds else (out, occ)
