"""ctypes binding of tests/first_available_fast.cpp, the brute-force restatement of profile alternatives (ISL_FLAG_FIRST_AVAILABLE,
include/islplace.h A1-A8) over flat occupancy bytes, every policy.

It is compiled with g++ into a fresh temporary directory once per process (the source tree may be read-only), so it needs no build step
of its own.  ``place`` takes the engine's inputs in canonical order and returns ``(records, occupancy after, placed)``.
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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "first_available_fast.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_first_available_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libfirst_available_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.fa_place.restype = u
        L.fa_place.argtypes = [u, p, u, u, p, p, p, p, u, u, u, u, u, u, p, p, u]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def place(node_off, rows, occ, requests, policy=E.POLICY_FIRST_FIT, quirks=E.QUIRKS_REF_EXACT, node_table=None, lo=0, hi=None,
          flagged=True, memo=False):
    """One batch (isl_place_batch on the partition [lo, hi), or isl_place_batch_range(lo, hi)).  ``rows``: [n_profiles] or
    [n_tables][n_profiles] with ``node_table`` [n_nodes]; ``flagged``: an ISL_FLAG_FIRST_AVAILABLE engine, else an unflagged one.
    ``memo``: the best-fit family's score of every (table, profile, byte) is walked once and remembered, which 2^20-GPU
    ISL_POLICY_MIN_FRAG calls need; off, every GPU is walked for every ALLOC (the one-core baseline of tools/first_available_time.py)."""
    node_off = np.ascontiguousarray(node_off, dtype=np.uint32)
    rows2 = np.ascontiguousarray(np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1]))
    n_nodes = len(node_off) - 1
    table = np.zeros(n_nodes, dtype=np.uint8) if node_table is None else np.ascontiguousarray(node_table, dtype=np.uint8)
    dsize = default_sizes(node_off, rows2, node_table)
    occ = np.array(occ, dtype=np.uint8)
    G = int(node_off[-1])
    assert len(occ) == G
    hi = G if hi is None else hi
    assert 0 <= lo <= hi <= G
    requests = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    placed = lib().fa_place(n_nodes, _ptr(node_off), rows2.shape[0], rows2.shape[1], _ptr(rows2), _ptr(table), _ptr(dsize), _ptr(occ),
                            lo, hi, quirks, policy, int(flagged), len(requests), _ptr(requests), _ptr(out), int(memo))
    return out, occ, int(placed)


def pods(groups, handles=None):
    """Requests of pods: ``groups`` is a list of profile-index lists, one per pod (its alternatives in order); a pod's requests carry its
    index as handle (or ``handles[i]``)."""
    n = sum(len(g) for g in groups)
    req = np.zeros(n, dtype=E.REQUEST_DTYPE)
    k = 0
    for i, g in enumerate(groups):
        for p in g:
            req[k] = (i if handles is None else handles[i], p, E.OP_ALLOC, 0, 0)
            k += 1
    return req
