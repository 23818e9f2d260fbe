"""Snapshot entry points without a GPU: the ctypes declarations of b2s.py follow include/b2s.h, and NULL arguments are refused with
B2S_E_INVALID before any CUDA call."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT, load_b2s

b2s = load_b2s()

FUNCS = ("b2s_band_save_state", "b2s_band_load_state", "b2s_recorder_bank_save_state", "b2s_recorder_bank_load_state")
CTYPES = {"b2s_band*": C.c_void_p, "b2s_recorder_bank*": C.c_void_p, "void*": C.c_void_p, "constvoid*": C.c_void_p, "size_t": C.c_size_t,
          "size_t*": C.POINTER(C.c_size_t)}


def declared(name):
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2s.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, f"{name} is not declared"
    return [re.sub(r"\s+", "", re.sub(r"\w+$", "", p.strip())) for p in m.group(1).split(",")]  # the types, without the names


def lib_or_skip():
    if not os.path.exists(b2s.LIB_PATH):
        pytest.skip("libb2s.so not built; run __graft_entry__.build()")
    return b2s.lib()


@pytest.mark.parametrize("name", FUNCS)
def test_binding_matches_the_header(name):
    params = declared(name)
    kind = "save" if name.endswith("save_state") else "load"
    assert params[1:] == (["void*", "size_t", "size_t*"] if kind == "save" else ["constvoid*", "size_t"]), params
    f = getattr(lib_or_skip(), name)
    assert f.argtypes == [CTYPES[p] for p in params] and f.restype == C.c_int
    owner = b2s.Band if name.startswith("b2s_band") else b2s.RecorderBank
    assert callable(getattr(owner, kind + "_state", None))


def test_null_arguments_are_refused_without_a_gpu():
    L = lib_or_skip()
    written = C.c_size_t(123)
    buf = (C.c_uint8 * 64)()
    for prefix in ("b2s_band", "b2s_recorder_bank"):
        save, load = getattr(L, prefix + "_save_state"), getattr(L, prefix + "_load_state")
        assert save(None, buf, 64, C.byref(written)) == -1
        assert save(None, None, 0, None) == -1
        assert load(None, buf, 64) == -1
        assert load(None, None, 0) == -1
        assert b"NULL" in L.b2s_last_error()
