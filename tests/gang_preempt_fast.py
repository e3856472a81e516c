"""ctypes binding of tests/gang_preempt_fast.cpp, the brute-force restatement of isl_preempt on an ISL_FLAG_GANG_PREEMPT engine (P1-P8).

It is compiled with g++ into a fresh temporary directory once per process (the source tree may be read-only), so it needs no build step
of its own.  ``preempt`` takes the engine's inputs in canonical order and returns ``(rc, results, evict)`` as isl_preempt would.
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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gang_preempt_fast.cpp")
_lib = None

PER_GANG = 4      # ``locality``: each gang's ALLOC ``start`` byte names it (an ISL_FLAG_GANG_LOCALITY engine)


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_gang_preempt_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libgang_preempt_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.gpf_preempt.restype = C.c_int
        L.gpf_preempt.argtypes = [u, u, p, p, p, p, u, p, u, u, u, u, u, u, p, p, u, p, p, p]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def preempt(node_off, rows, occ, requests, priority, victims, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT, node_table=None,
            lo=0, hi=None, locality=0):
    """``rows``: [n_profiles] or [n_tables][n_profiles] with ``node_table`` [n_nodes]; [lo, hi): the canonical partition; ``locality``:
    E.GANG_ANY_NODES, _ONE_NODE or _DISTINCT_NODES for every gang, or PER_GANG.  Gangs are the runs of equal ``handle``."""
    node_off = np.ascontiguousarray(node_off, dtype=np.uint32)
    rows2 = np.ascontiguousarray(np.asarray(rows, dtype=E.PROFILE_DTYPE).reshape(-1, np.asarray(rows).shape[-1]))
    G = int(node_off[-1])
    hi = G if hi is None else hi
    gtab = np.zeros(G, dtype=np.uint8)
    if node_table is not None:
        for n, t in enumerate(node_table):
            gtab[node_off[n]:node_off[n + 1]] = t
    dsize = default_sizes(node_off, rows2, node_table)
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    requests = np.ascontiguousarray(requests, dtype=E.REQUEST_DTYPE)
    priority = np.ascontiguousarray(priority, dtype=np.uint8)
    victims = np.ascontiguousarray(victims, dtype=E.VICTIM_DTYPE)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    evict = np.zeros((len(requests), 8), dtype=np.uint32)
    rc = lib().gpf_preempt(G, rows2.shape[1], _ptr(rows2), _ptr(gtab), _ptr(dsize), _ptr(occ), len(node_off) - 1, _ptr(node_off), lo, hi,
                           quirks, policy, locality, len(requests), _ptr(requests), _ptr(priority), len(victims), _ptr(victims), _ptr(out),
                           _ptr(evict))
    return rc, out, evict
