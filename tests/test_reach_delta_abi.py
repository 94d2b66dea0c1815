"""CPU-side checks of B200_reach_batch_delta: argument and dimension errors come back before any device work, host-resident
operands are refused, and without a GPU the call fails loudly (there is no CPU fallback).  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, I64, P
from falkordb_b200.grb import Matrix


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def reach_delta(src, ms, dps, dms, nops=None, reached=True):
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    h, lv = P(), I64()
    src = np.ascontiguousarray(src, dtype=np.uint64)
    return lib().B200_reach_batch_delta(C.byref(h) if reached else None, src.ctypes.data if len(src) else None, len(src),
                                        None if ms is None else arr(ms), None if dps is None else arr(dps),
                                        None if dms is None else arr(dms), len(ms or ()) if nops is None else nops, 2, 0,
                                        C.byref(lv))


def test_null_pointers():
    fb.init()
    m = Matrix(16, 16)
    assert reach_delta([0, 1], [m], None, None, reached=False) == -2      # GrB_NULL_POINTER: reached
    assert reach_delta([0, 1], None, None, None, nops=1) == -2            # m
    assert reach_delta([0, 1], [None], None, None) == -2                  # m[0]
    h, lv = P(), I64()
    ms = (C.c_void_p * 1)(m.h)
    assert lib().B200_reach_batch_delta(C.byref(h), None, 2, ms, None, None, 1, 2, 0, C.byref(lv)) == -2   # sources


def test_operand_count_and_dimensions():
    fb.init()
    m, d, small, rect = Matrix(16, 16), Matrix(16, 16), Matrix(8, 8), Matrix(16, 8)
    assert reach_delta([0], [m], None, None, nops=0) == -3                # GrB_INVALID_VALUE: nops < 1
    assert reach_delta([0], [m], None, None, nops=-1) == -3
    assert reach_delta([0], [rect], None, None) == -6                     # GrB_DIMENSION_MISMATCH: not square
    assert reach_delta([0], [m, small], None, None) == -6                 # operands of different sizes
    assert reach_delta([0], [m], [small], None) == -6                     # dp not shaped like m
    assert reach_delta([0], [m], None, [small]) == -6                     # dm not shaped like m
    assert reach_delta([0], [m, m], [d, None], [None, rect]) == -6


def test_host_resident_operands_are_refused():
    n = 1 << 60
    m = Matrix(n, n)
    assert reach_delta([0], [m], None, None) == -8                        # GrB_NOT_IMPLEMENTED
    assert reach_delta([0], [m], [Matrix(n, n)], [None]) == -8


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_reach_delta_fails_loudly_without_gpu():
    fb.init()
    m, dp, dm = Matrix(16, 16), Matrix(16, 16), Matrix(16, 16)
    m.set(0, 1)
    dp.set(1, 2)
    dm.set(0, 1)
    assert reach_delta([0], [m], [dp], [dm]) == -7002                     # GxB_GPU_ERROR
    assert reach_delta([0], [m], None, None) == -7002
    with pytest.raises(fb.GrbError) as e:
        fb.reach_batch([0], [m, m], 2, deltas=[(dp, dm), (None, None)])
    assert e.value.info == -7002
