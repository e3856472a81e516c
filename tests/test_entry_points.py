"""Every C-ABI entry point of islplace.cu that takes an engine opens with one Entry, the guard that takes the engine lock, checks the
engine state and makes the engine's device current; the state it asks for (Needs) is the one its row in tests/engine_contract.py
refuses without.  These checks read the source; they need no GPU."""
import ctypes as C
import re

import numpy as np
import pytest

import engine_contract as K
from instaslice_b200 import engine as E
from test_engine_ownership import _body, _code

# the engine states each Needs value refuses with ISL_ESTATE (Needs::open_stream: every idle state)
REFUSED = {"nothing": set(), "profiles": {"created", "inventory"}, "inventory": {"created", "profiles"},
           "ready": {"created", "profiles", "inventory"}, "open_stream": set(K.STATES)}
# outside the guard: the lock-free isl_stream_wait, destroy (it closes an open stream first) and the calls that read no engine state
EXEMPT = (K.LEGAL_DURING_OPEN | K.NO_ENGINE) - {"isl_stream_submit", "isl_stream_close"}
DEBUG_ONLY = {"isl_debug_spec_rounds"}          # a debugging aid outside include/islplace.h: no contract row


def _definitions(code):
    return set(re.findall(r"^\S[^\n;]*?\b(isl_\w+)\([^;{]*\)\s*\{", code, flags=re.M))


def test_every_entry_point_takes_the_guard_its_contract_row_names():
    code = _code()
    names = _definitions(code)
    assert names == set(K.CODES) | DEBUG_ONLY, names ^ (set(K.CODES) | DEBUG_ONLY)
    for name in sorted(names):
        needs = re.findall(r"\bEntry\s+\w+\(\s*e\s*,\s*Needs::(\w+)", _body(code, name))
        if name in EXEMPT:
            assert needs == [], name
            continue
        assert len(needs) == 1, (name, needs)
        if name in DEBUG_ONLY:
            continue
        refused = {s for s in K.STATES if K.expected(name, s, K.Ctx(snapshot=True)) == E.ESTATE}
        assert REFUSED[needs[0]] == refused, (name, needs[0], refused)


def test_lock_and_readiness_only_in_the_guard():
    code = _code()
    guard = _body(code, "Entry")
    rest = code.replace(guard, "")
    assert "e->mu" in guard and "->mu" not in rest
    for flag in ("have_profiles", "have_inventory"):
        assert flag in guard
        uses = re.findall(r"\b%s\b(\s*=(?!=))?" % flag, rest)
        assert uses and all(uses), flag           # declared and set, never read


@pytest.mark.gpu
@pytest.mark.parametrize("policy", [E.POLICY_BEST_FIT, E.POLICY_RIGHT_TO_LEFT])
def test_empty_partitioned_call_returns_ok_before_the_policy_check(policy):
    """Best-fit and right-to-left engines do not partition (ISL_EINVAL), but an empty partitioned call has nothing to place and returns
    ISL_OK first.  Needs an H100."""
    import torch
    from instaslice_b200 import tables
    eng = E.Engine(max_gpus=64, max_batch=64, policy=policy)
    eng.load_profiles(E.make_profiles(tables.H100_80GB))
    eng.load_inventory(np.array([0, 8], dtype=np.uint32), np.zeros(8, dtype=np.uint8))
    buf = torch.zeros(64 * 8, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    L, h, p = eng._lib, eng._h, C.c_void_p(buf.data_ptr())
    for n, want in ((0, E.OK), (8, E.EINVAL)):
        sizes = np.array([n], dtype=np.uint32)
        assert L.isl_place_batch_partitioned(h, n, p, p, None, p) == want, n
        assert L.isl_place_stream_partitioned(h, 1, sizes.ctypes.data_as(C.c_void_p), p, p, 1) == want, n
    eng.close()
