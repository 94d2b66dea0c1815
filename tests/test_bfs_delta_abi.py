"""CPU-side checks of B200_bfs_delta: argument, dimension and index errors come back before any device work, host-resident operands
are refused, and without a GPU the call fails loudly (there is no CPU fallback).  No kernel is launched here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib
from falkordb_b200.grb import Matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def bfs_delta(ms, dps, dms, src=0, dest=-1, nops=None, level=True):
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    n = 16
    lv = np.empty(n, np.int64)
    pr = np.empty(n, np.int64)
    return lib().B200_bfs_delta(None if ms is None else arr(ms), None if dps is None else arr(dps), None if dms is None else arr(dms),
                                len(ms or ()) if nops is None else nops, src, -1, dest, lv.ctypes.data if level else None,
                                pr.ctypes.data, 0, None)


def test_null_pointers():
    fb.init()
    m = Matrix(16, 16)
    assert bfs_delta(None, None, None, nops=1) == -2                      # GrB_NULL_POINTER: m
    assert bfs_delta([None], None, None) == -2                            # m[0]
    assert bfs_delta([m], None, None, level=False) == -2                  # level


def test_operand_count_and_dimensions():
    fb.init()
    m, d, small, rect = Matrix(16, 16), Matrix(16, 16), Matrix(8, 8), Matrix(16, 8)
    assert bfs_delta([m], None, None, nops=0) == -3                       # GrB_INVALID_VALUE: nops < 1
    assert bfs_delta([m], None, None, nops=-1) == -3
    assert bfs_delta([rect], None, None) == -6                            # GrB_DIMENSION_MISMATCH: not square
    assert bfs_delta([m, small], None, None) == -6                        # operands of different sizes
    assert bfs_delta([m], [small], None) == -6                            # dp not shaped like m
    assert bfs_delta([m], None, [small]) == -6                            # dm not shaped like m
    assert bfs_delta([m, m], [d, None], [None, rect]) == -6


def test_source_and_destination_out_of_range():
    fb.init()
    m = Matrix(16, 16)
    assert bfs_delta([m], None, None, src=16) == -4                       # GrB_INVALID_INDEX
    assert bfs_delta([m], None, None, src=0, dest=16) == -4
    assert bfs_delta([m, m], [None, None], [None, None], src=1 << 40) == -4


def test_host_resident_operands_are_refused():
    n = 1 << 60
    m = Matrix(n, n)
    assert bfs_delta([m], None, None) == -8                               # GrB_NOT_IMPLEMENTED
    assert bfs_delta([m], [Matrix(n, n)], [None]) == -8


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_bfs_delta_fails_loudly_without_gpu():
    fb.init()
    m, dp, dm = Matrix(16, 16), Matrix(16, 16), Matrix(16, 16)
    m.set(0, 1)
    dp.set(1, 2)
    dm.set(0, 1)
    assert bfs_delta([m], [dp], [dm]) == -7002                            # GxB_GPU_ERROR
    assert bfs_delta([m], None, None) == -7002
    with pytest.raises(fb.GrbError) as e:
        fb.bfs([m, m], 0, deltas=[(dp, dm), (None, None)])
    assert e.value.info == -7002


def test_symbol_is_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "falkordb_b200", "libb200grb.so")], capture_output=True,
                         text=True, check=True).stdout
    assert any(line.split()[-1] == "B200_bfs_delta" for line in out.splitlines() if line.strip())
