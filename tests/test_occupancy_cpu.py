"""Spectrum occupancy without a GPU: the ctypes declarations follow include/b2s.h, and NULL or bad arguments are refused before any
CUDA call."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT, load_b2s

b2s = load_b2s()


def declared(name):
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b2s.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", header)
    assert m, f"{name} is not declared"
    return [re.sub(r"\s+", "", re.sub(r"\w+$", "", p.strip())) for p in m.group(1).split(",")]


def lib_or_skip():
    if not os.path.exists(b2s.LIB_PATH):
        pytest.skip("libb2s.so not built; run __graft_entry__.build()")
    return b2s.lib()


def test_bindings_match_the_header():
    assert declared("b2s_band_set_occupancy") == ["b2s_band*", "int"]
    assert declared("b2s_band_occupancy_centers") == ["b2s_band*", "int32_t*", "int", "int*"]
    assert declared("b2s_band_get_occupancy") == ["b2s_band*", "int32_t", "uint32_t*", "uint32_t*", "float*", "int64_t*", "int64_t*", "int64_t*", "int"]
    L = lib_or_skip()
    assert L.b2s_band_set_occupancy.argtypes == [C.c_void_p, C.c_int] and L.b2s_band_set_occupancy.restype == C.c_int
    f = L.b2s_band_occupancy_centers
    assert f.argtypes == [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)] and f.restype == C.c_int
    f = L.b2s_band_get_occupancy
    i64 = C.POINTER(C.c_int64)
    assert f.argtypes == [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, i64, i64, i64, C.c_int] and f.restype == C.c_int
    for name in ("set_occupancy", "occupancy_centers", "occupancy"):
        assert callable(getattr(b2s.Band, name, None)), name
    assert b2s.Occupancy._fields == ("above_start", "above_stop", "max_db", "frames", "detect_frames", "truncated")


def test_null_and_bad_arguments_are_refused():
    L = lib_or_skip()
    n = 16
    a, s, m = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.float32)
    frames, detect, trunc = C.c_int64(5), C.c_int64(6), C.c_int64(7)
    count = C.c_int(9)
    centres = np.zeros(4, np.int32)
    ptr = lambda x: x.ctypes.data_as(C.c_void_p)
    assert L.b2s_band_set_occupancy(None, 1) == -1
    assert L.b2s_band_set_occupancy(None, 0) == -1
    assert L.b2s_band_occupancy_centers(None, ptr(centres), 4, C.byref(count)) == -1
    assert L.b2s_band_occupancy_centers(None, None, 0, None) == -1
    assert L.b2s_band_get_occupancy(None, 100_000_000, ptr(a), ptr(s), ptr(m), C.byref(frames), C.byref(detect), C.byref(trunc), 0) == -1
    assert L.b2s_band_get_occupancy(None, 100_000_000, None, None, None, None, None, None, 1) == -1
    assert count.value == 9 and (frames.value, detect.value, trunc.value) == (5, 6, 7)
    assert b"NULL" in L.b2s_last_error()
