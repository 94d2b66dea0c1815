"""CPU-side checks of the dirty-hop entries B200_Matrix_delta_lmxm and B200_traverse_batch_delta: argument and dimension errors
come back before any device work, and without a GPU both fail loudly (there is no CPU fallback).  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Matrix


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def traverse_delta(src, hops, dps, dms, out_p, out_j):
    arr = lambda ms: (C.c_void_p * len(ms))(*[None if m is None else m.h for m in ms])
    nv, fl, fmt = U64(0), U64(0), C.c_int(0)
    src = np.ascontiguousarray(src, dtype=np.uint64)
    return lib().B200_traverse_batch_delta(src.ctypes.data, len(src), arr(hops), None if dps is None else arr(dps),
                                           None if dms is None else arr(dms), len(hops), fb.OUT_CSR, None, 0, out_p.ctypes.data,
                                           out_j.ctypes.data, len(out_j), C.byref(nv), C.byref(fl), C.byref(fmt))


def test_delta_lmxm_null_and_dimension_errors():
    fb.init()
    L = lib()
    F, m, d, small = Matrix(4, 16), Matrix(16, 16), Matrix(16, 16), Matrix(8, 8)
    assert L.B200_Matrix_delta_lmxm(None, m.h, d.h, d.h) == -2           # GrB_NULL_POINTER
    assert L.B200_Matrix_delta_lmxm(F.h, None, d.h, d.h) == -2
    assert L.B200_Matrix_delta_lmxm(F.h, small.h, None, None) == -6      # GrB_DIMENSION_MISMATCH: F * m does not fit F
    assert L.B200_Matrix_delta_lmxm(F.h, m.h, small.h, None) == -6       # dp not shaped like m
    assert L.B200_Matrix_delta_lmxm(F.h, m.h, None, small.h) == -6       # dm not shaped like m
    assert L.B200_Matrix_delta_lmxm(Matrix(4, 8).h, m.h, d.h, None) == -6


def test_traverse_batch_delta_null_and_dimension_errors():
    fb.init()
    m, d, small = Matrix(16, 16), Matrix(16, 16), Matrix(8, 8)
    p, j = np.zeros(3, np.uint64), np.zeros(8, np.uint32)
    L = lib()
    nv, fl, fmt = U64(0), U64(0), C.c_int(0)
    assert L.B200_traverse_batch_delta(None, 2, None, None, None, 1, fb.OUT_CSR, None, 0, p.ctypes.data, j.ctypes.data, 8,
                                       C.byref(nv), C.byref(fl), C.byref(fmt)) == -2
    assert traverse_delta([0, 1], [m], [small], None, p, j) == -6
    assert traverse_delta([0, 1], [m], [None], [small], p, j) == -6
    assert traverse_delta([0, 1], [m, small], [d, None], None, p, j) == -6


def test_host_resident_operands_are_refused():
    n = 1 << 60
    F, m = Matrix(4, n), Matrix(n, n)
    assert lib().B200_Matrix_delta_lmxm(F.h, m.h, m.h, None) == -8        # GrB_NOT_IMPLEMENTED


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_delta_entries_fail_loudly_without_gpu():
    fb.init()
    F, m, dp, dm = Matrix(4, 16), Matrix(16, 16), Matrix(16, 16), Matrix(16, 16)
    m.set(0, 1)
    dp.set(1, 2)
    with pytest.raises(fb.GrbError) as e:
        F.delta_lmxm_fused(m, dp, dm)
    assert e.value.info == -7002
    p, j = np.zeros(3, np.uint64), np.zeros(8, np.uint32)
    assert traverse_delta([0, 1], [m], [dp], [dm], p, j) == -7002
