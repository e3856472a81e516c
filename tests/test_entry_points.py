"""Every C-ABI entry point of islplace.cu that takes an engine opens with one Entry, the guard that takes the engine lock, checks the
engine state and makes the engine's device current; the state it asks for (Needs) is the one its row in tests/engine_contract.py
refuses without.  These checks read the source; they need no GPU."""
import re

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
