"""CPU-side checks of the union-hop entries B200_Matrix_union_lmxm and B200_traverse_batch_union: argument and dimension errors
come back before any device work, host-resident operands are refused, and without a GPU the calls fail loudly (there is no CPU
fallback).  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Matrix


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def arr(xs):
    return (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])


def union_lmxm(F, ms, dps, dms, nops=None):
    return lib().B200_Matrix_union_lmxm(None if F is None else F.h, None if ms is None else arr(ms),
                                        None if dps is None else arr(dps), None if dms is None else arr(dms),
                                        len(ms or ()) if nops is None else nops)


def traverse_union(src, nops, union, ms, dps=None, dms=None, nhops=None):
    src = np.ascontiguousarray(src, dtype=np.uint64)
    p, j = np.zeros(len(src) + 1, np.uint64), np.zeros(64, np.uint32)
    nv, fl, ch = U64(0), U64(0), C.c_int(0)
    ints = lambda xs: None if xs is None else (C.c_int * max(1, len(xs)))(*xs)
    return lib().B200_traverse_batch_union(src.ctypes.data if len(src) else None, len(src), ints(nops), ints(union),
                                           len(nops or ()) if nhops is None else nhops, None if ms is None else arr(ms),
                                           None if dps is None else arr(dps), None if dms is None else arr(dms), fb.OUT_CSR, None, 0,
                                           p.ctypes.data, j.ctypes.data, len(j), C.byref(nv), C.byref(fl), C.byref(ch))


def test_null_pointers():
    fb.init()
    F, m = Matrix(4, 16), Matrix(16, 16)
    assert union_lmxm(None, [m], None, None) == -2                        # GrB_NULL_POINTER: F
    assert union_lmxm(F, None, None, None, nops=1) == -2                  # m
    assert union_lmxm(F, [None], None, None) == -2                        # m[0]
    assert traverse_union([0], None, [1], [m]) == -2                      # hop_nops
    assert traverse_union([0], [1], None, [m]) == -2                      # hop_union
    assert traverse_union([0], [1], [1], None, nhops=1) == -2             # m
    assert traverse_union([0], [2], [1], [m, None]) == -2                 # m[1]
    ms = (C.c_void_p * 1)(m.h)
    one = (C.c_int * 1)(1)
    p, j = np.zeros(3, np.uint64), np.zeros(8, np.uint32)
    assert lib().B200_traverse_batch_union(None, 2, one, one, 1, ms, None, None, fb.OUT_CSR, None, 0, p.ctypes.data, j.ctypes.data,
                                           8, None, None, None) == -2     # sources


def test_operand_count_and_dimensions():
    fb.init()
    F, m, d, small, rect = Matrix(4, 16), Matrix(16, 16), Matrix(16, 16), Matrix(8, 8), Matrix(16, 8)
    assert union_lmxm(F, [m], None, None, nops=0) == -3                   # GrB_INVALID_VALUE: nops < 1
    assert union_lmxm(F, [m], None, None, nops=-1) == -3
    assert union_lmxm(F, [rect], None, None) == -6                        # GrB_DIMENSION_MISMATCH: not square
    assert union_lmxm(F, [m, small], None, None) == -6                    # operands of different sizes
    assert union_lmxm(F, [m], [small], None) == -6                        # dp not shaped like m
    assert union_lmxm(F, [m], None, [small]) == -6                        # dm not shaped like m
    assert union_lmxm(F, [m, m], [d, None], [None, rect]) == -6
    assert union_lmxm(Matrix(4, 8), [m], None, None) == -6                # F * m does not fit F
    assert traverse_union([0], [0], [1], [m]) == -3                       # a hop without operands
    assert traverse_union([0], [1], [1], [m], nhops=0) == -3              # nhops < 1
    assert traverse_union([0], [2], [0], [m, m]) == -3                    # a delta hop takes one operand
    assert traverse_union([0], [1, 2], [0, 0], [m, m, m]) == -3
    assert traverse_union([0], [1, 1], [0, 1], [m, small]) == -6          # hops of different sizes
    assert traverse_union([0], [2], [1], [m, rect]) == -6
    assert traverse_union([0], [1], [1], [m], [None], [small]) == -6


def test_host_resident_operands_are_refused():
    n = 1 << 60
    m, F = Matrix(n, n), Matrix(4, n)
    assert union_lmxm(F, [m], None, None) == -8                           # GrB_NOT_IMPLEMENTED
    assert union_lmxm(F, [m, m], [Matrix(n, n), None], None) == -8
    assert traverse_union([0], [1], [1], [m]) == -8
    assert traverse_union([0], [1], [0], [m]) == -8                       # a delta hop of the union entry too


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_union_hop_fails_loudly_without_gpu():
    fb.init()
    m, dp, dm = Matrix(16, 16), Matrix(16, 16), Matrix(16, 16)
    m.set(0, 1)
    dp.set(1, 2)
    dm.set(0, 1)
    F = Matrix(1, 16)
    F.set(0, 0)
    assert union_lmxm(F, [m, m], [dp, None], [dm, None]) == -7002         # GxB_GPU_ERROR
    assert union_lmxm(F, [m], None, None) == -7002
    assert traverse_union([0], [2], [1], [m, m], [dp, None], [dm, None]) == -7002
    assert traverse_union([0], [1, 1], [0, 1], [m, m]) == -7002
    with pytest.raises(fb.GrbError) as e:
        fb.traverse_batch([0], [[m, m]], fb.OUT_CSR, out_p=np.zeros(2, np.uint64), out_j=np.zeros(8, np.uint32),
                          deltas=[[(dp, dm), (None, None)]])
    assert e.value.info == -7002
    with pytest.raises(fb.GrbError) as e:
        F.union_lmxm([m], [(dp, dm)])
    assert e.value.info == -7002
