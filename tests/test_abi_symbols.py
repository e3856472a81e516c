"""The C-ABI library loads on a CPU-only box and exports every symbol include/islplace.h declares."""
import ctypes
import os
import re

from instaslice_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "islplace.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(isl_[a-z_]+)\s*\(", text)))


def test_header_and_signatures_agree():
    assert declared_symbols() == sorted(E.SIGNATURES)


def test_every_signature_has_a_contract_row():
    """Every entry point is classified in tests/engine_contract.py: its code in every engine state, and whether an open stream allows it.
    A symbol added to the ABI fails here until it has a row."""
    import engine_contract as K
    assert sorted(K.CODES) == sorted(E.SIGNATURES)
    assert K.LEGAL_DURING_OPEN <= set(E.SIGNATURES) and K.NO_ENGINE <= set(E.SIGNATURES)
    contexts = [K.Ctx(policy, flags, empty, snap) for policy in range(4) for flags in (0, E.FLAG_ALL_NODES)
                for empty in (False, True) for snap in (False, True)]
    for name, row in K.CODES.items():
        assert set(row) == set(K.ALL_STATES), name
        for ctx in contexts:
            for state in K.ALL_STATES:
                code = K.expected(name, state, ctx)
                assert code in (K.VALUE, E.OK, E.EINVAL, E.ESTATE, E.ERANGE), (name, state, code)
            if name in K.LEGAL_DURING_OPEN or name in K.NO_ENGINE:
                continue
            # refused in every sub-state of an open stream; only a config the call never accepts reports EINVAL first
            never = {K.expected(name, s, ctx) for s in K.STATES} == {E.EINVAL}
            for state in K.OPEN_STATES:
                assert K.expected(name, state, ctx) == (E.EINVAL if never else E.ESTATE), (name, state, ctx)


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(E.LIB_PATH)
    for name in declared_symbols():
        assert hasattr(lib, name), name


def test_record_layouts_match_header():
    assert E.REQUEST_DTYPE.itemsize == 8 and E.RESULT_DTYPE.itemsize == 8 and E.SPAN_DTYPE.itemsize == 8
    assert E.PROFILE_DTYPE.itemsize == 24
    assert ctypes.sizeof(E.Config) == 32
    lib = E.load_library()
    assert lib.isl_abi_version() == E.ABI_VERSION
    assert lib.isl_strerror(E.EINVAL).decode().startswith("invalid")


def test_argument_validation_without_gpu():
    """Pure argument checks return before any CUDA call."""
    lib = E.load_library()
    h = ctypes.c_void_p()
    bad = E.Config(99, 0, 3, -1, 16, 16, 0, 0)          # wrong ABI version
    assert lib.isl_create(ctypes.byref(bad), ctypes.byref(h)) == E.EINVAL
    bad = E.Config(E.ABI_VERSION, 0, 3, -1, 0, 16, 0, 0)  # zero capacity
    assert lib.isl_create(ctypes.byref(bad), ctypes.byref(h)) == E.EINVAL
    bad = E.Config(E.ABI_VERSION, 0, 3, -1, (1 << 24) + 1, 16, 0, 0)
    assert lib.isl_create(ctypes.byref(bad), ctypes.byref(h)) == E.EINVAL
    bad = E.Config(E.ABI_VERSION, 0, 0xF0, -1, 16, 16, 0, 0)   # unknown quirk bits
    assert lib.isl_create(ctypes.byref(bad), ctypes.byref(h)) == E.EINVAL
    assert lib.isl_destroy(None) == E.EINVAL
    assert lib.isl_num_gpus(None) == 0


def test_header_is_plain_c99(tmp_path):
    """What cgo includes must be C, not C++: the header alone compiles with gcc -std=c99 -pedantic."""
    import shutil
    import subprocess
    if not shutil.which("gcc"):
        import pytest
        pytest.skip("no gcc")
    src = tmp_path / "t.c"
    src.write_text('#include "islplace.h"\nint main(void) { isl_config c; isl_request r; isl_result s; (void)c; (void)r; (void)s; return 0; }\n')
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), "-c", str(src), "-o",
                    str(tmp_path / "t.o")], check=True)


def test_no_gpu_means_error_not_fallback():
    """Without a GPU isl_create fails with ISL_ECUDA — there is no CPU path behind the ABI."""
    import torch
    if torch.cuda.is_available():
        import pytest
        pytest.skip("a GPU is present")
    lib = E.load_library()
    h = ctypes.c_void_p()
    ok = E.Config(E.ABI_VERSION, 0, 3, -1, 16, 16, 0, 0)
    assert lib.isl_create(ctypes.byref(ok), ctypes.byref(h)) == E.ECUDA
