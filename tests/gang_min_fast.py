"""ctypes binding of tests/gang_min_fast.cpp, the brute-force restatement of isl_place_gangs on an ISL_FLAG_GANG_MIN_MEMBERS engine over
flat occupancy bytes, for all four localities.

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

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gang_min_fast.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="isl_gang_min_fast_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libgang_min_fast.so")
        subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-o", so, _SRC], check=True)
        L = C.CDLL(so)
        p, u = C.c_void_p, C.c_uint32
        L.gmf_place_gangs.restype = C.c_uint64
        L.gmf_place_gangs.argtypes = [u, p, p, u, p, p, p, u, u, u, u, u, p, p, p, u, p, p]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def effective_minimum(requests, gang_off) -> np.ndarray:
    """m' of every gang (M1) from the ``size`` byte of its ALLOC members: k when m = 0 or m >= k, else m (0 for a gang without ALLOCs).
    Raises ValueError when two ALLOC members of a gang carry different bytes (M6)."""
    out = np.zeros(len(gang_off) - 1, dtype=np.uint32)
    for i, (a, b) in enumerate(zip(gang_off[:-1], gang_off[1:])):
        sizes = requests["size"][a:b][requests["op"][a:b] == E.OP_ALLOC]
        if len(set(sizes.tolist())) > 1:
            raise ValueError(f"gang {i}: ALLOC members carry different minima")
        k, m = len(sizes), int(sizes[0]) if len(sizes) else 0
        out[i] = k if m == 0 or m >= k else m
    return out


def place_gangs(node_off, rows, occ, requests, gang_off, locality, quirks=E.QUIRKS_REF_EXACT, policy=E.POLICY_FIRST_FIT,
                node_table=None, lo=0, hi=None, memo=True, min_members=None):
    """``locality``: one ``E.GANG_*`` per gang, or one value for every gang; ``min_members``: m' per gang, by default
    ``effective_minimum`` of the requests' ``size`` bytes.  ``rows``: [n_profiles] or [n_tables][n_profiles] with ``node_table``
    [n_nodes]; [lo, hi): the engine's partition (canonical); ``memo``: ISL_POLICY_MIN_FRAG scores are walked once per (table, profile,
    byte) and remembered."""
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
    loc = np.ascontiguousarray(np.broadcast_to(np.asarray(locality, dtype=np.uint8), (n_gangs,)))
    mins = effective_minimum(requests, gang_off) if min_members is None else np.ascontiguousarray(min_members, dtype=np.uint32)
    out = np.zeros(len(requests), dtype=E.RESULT_DTYPE)
    placed = lib().gmf_place_gangs(n_nodes, _ptr(node_off), _ptr(table), rows2.shape[1], _ptr(rows2), _ptr(dsize), _ptr(occ), lo, hi,
                                   quirks, policy, n_gangs, _ptr(gang_off), _ptr(requests), _ptr(out), int(memo), _ptr(loc), _ptr(mins))
    return out, occ, int(placed)
