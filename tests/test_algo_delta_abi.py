"""CPU-side checks of B200_adjacency_delta: argument, dimension and index errors come back before any device work, host-resident
operands are refused, and without a GPU the call fails loudly (there is no CPU fallback).  No kernel is launched here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, P
from falkordb_b200.grb import Matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def adjacency(ms, dps=None, dms=None, n_out=16, keep=None, nkeep=None, nops=None, out=True, symmetric=0):
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    kp = None if keep is None else np.ascontiguousarray(keep, np.uint64)
    h = P()
    return lib().B200_adjacency_delta(C.byref(h) if out else None, None if ms is None else arr(ms), None if dps is None else arr(dps),
                                      None if dms is None else arr(dms), len(ms or ()) if nops is None else nops, n_out,
                                      None if kp is None else kp.ctypes.data, (0 if kp is None else len(kp)) if nkeep is None else nkeep,
                                      symmetric)


def test_null_pointers():
    fb.init()
    m = Matrix(16, 16)
    assert adjacency([m], out=False) == -2                                # GrB_NULL_POINTER: A
    assert adjacency(None, nops=1) == -2                                  # m
    assert adjacency([None]) == -2                                        # m[0]


def test_operand_count_and_dimensions():
    fb.init()
    m, d, small, rect = Matrix(16, 16), Matrix(16, 16), Matrix(8, 8), Matrix(16, 8)
    assert adjacency([m], nops=0) == -3                                   # GrB_INVALID_VALUE: nops < 1
    assert adjacency([m], nops=-1) == -3
    assert adjacency([rect]) == -6                                        # GrB_DIMENSION_MISMATCH: not square
    assert adjacency([m, small]) == -6                                    # operands of different sizes
    assert adjacency([m], [small], None) == -6                            # dp not shaped like m
    assert adjacency([m], None, [small]) == -6                            # dm not shaped like m
    assert adjacency([m, m], [d, None], [None, rect]) == -6


def test_keep_list_errors():
    fb.init()
    m = Matrix(16, 16)
    assert adjacency([m], keep=[0, 3, 16]) == -4                          # GrB_INVALID_INDEX: id out of range
    assert adjacency([m], keep=[1 << 40]) == -4
    assert adjacency([m], keep=[2, 2, 5]) == -4                           # not strictly ascending
    assert adjacency([m], keep=[5, 3]) == -4
    assert adjacency([m, m], [None, None], [None, None], keep=[0, 15, 7]) == -4


def test_identity_form_needs_32_bit_ids():
    fb.init()
    m = Matrix(16, 16)
    assert adjacency([m], n_out=1 << 32) == -3                            # GrB_INVALID_VALUE: n_out >= 2^32


def test_host_resident_operands_are_refused():
    n = 1 << 60
    m = Matrix(n, n)
    assert adjacency([m]) == -8                                           # GrB_NOT_IMPLEMENTED
    assert adjacency([m], [Matrix(n, n)], [None]) == -8


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_adjacency_fails_loudly_without_gpu():
    fb.init()
    m, dp, dm = Matrix(16, 16), Matrix(16, 16), Matrix(16, 16)
    m.set(0, 1)
    dp.set(1, 2)
    dm.set(0, 1)
    assert adjacency([m], [dp], [dm]) == -7002                            # GxB_GPU_ERROR
    assert adjacency([m], keep=[0, 1, 2], symmetric=1) == -7002
    assert adjacency([m], keep=[]) == -7002
    with pytest.raises(fb.GrbError) as e:
        fb.adjacency([m, m], deltas=[(dp, dm), (None, None)], symmetric=True)
    assert e.value.info == -7002


def test_symbol_is_exported():
    out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "falkordb_b200", "libb200grb.so")], capture_output=True,
                         text=True, check=True).stdout
    assert any(line.split()[-1] == "B200_adjacency_delta" for line in out.splitlines() if line.strip())
    host = subprocess.run(["nm", "-D", "--defined-only", os.path.join(ROOT, "falkordb_b200", "libfdbhost.so")], capture_output=True,
                          text=True, check=True).stdout
    names = {line.split()[-1] for line in host.splitlines() if line.strip()}
    assert {"fdbh_algo_pagerank", "fdbh_algo_wcc", "fdbh_algo_cdlp"} <= names
