"""ctypes binding of tests/bestfit_fast.cpp, the brute-force restatement of k_bestfit over flat occupancy bytes: isl_place_batch (and
isl_place_batch_range) on an ISL_POLICY_BEST_FIT / _MIN_FRAG engine, and isl_place_gangs on an engine without a gang flag, every policy.

It is compiled with g++ into a fresh temporary directory once per process (the source tree may be read-only), so it needs no build step
of its own.  ``place`` and ``place_gangs`` take the engine's inputs in canonical order and return ``(records, occupancy after)``.
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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "bestfit_fast.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_bestfit_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libbestfit_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.bff_place_gangs.restype = None
        L.bff_place_gangs.argtypes = [u, u, p, p, p, p, u, u, u, u, u, p, p, p, u]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def place_gangs(node_off, rows, occ, requests, gang_off, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
                lo=0, hi=None, memo=True):
    """``rows``: [n_profiles] or [n_tables][n_profiles] with ``node_table`` [n_nodes]; [lo, hi): the engine's partition (canonical);
    ``memo``: every (table, profile, byte) is evaluated once and remembered, which 2^20-GPU ISL_POLICY_MIN_FRAG calls need."""
    node_off = np.asarray(node_off, dtype=np.int64)
    rows2 = np.ascontiguousarray(np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1]))
    n_nodes = len(node_off) - 1
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.asarray(node_table, dtype=np.uint8)
    gtab = np.ascontiguousarray(np.repeat(table, np.diff(node_off)))
    dsize = default_sizes(node_off, rows2, node_table)
    occ = np.array(occ, dtype=np.uint8)
    G = len(occ)
    assert G == int(node_off[-1])
    hi = G if hi is None else hi
    assert 0 <= lo <= hi <= G
    requests = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    gang_off = np.ascontiguousarray(gang_off, dtype=np.uint32)
    assert int(gang_off[-1]) == len(requests)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    lib().bff_place_gangs(G, rows2.shape[1], _ptr(rows2), _ptr(gtab), _ptr(dsize), _ptr(occ), lo, hi, quirks, policy, len(gang_off) - 1,
                          _ptr(gang_off), _ptr(requests), _ptr(out), int(memo))
    return out, occ


def place(node_off, rows, occ, requests, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_BEST_FIT, node_table=None, lo=0, hi=None,
          memo=True):
    """One batch (isl_place_batch on the partition [lo, hi), or isl_place_batch_range(lo, hi)): gangs of one."""
    return place_gangs(node_off, rows, occ, requests, np.arange(len(requests) + 1, dtype=np.uint32), quirks, policy, node_table, lo, hi,
                       memo)
