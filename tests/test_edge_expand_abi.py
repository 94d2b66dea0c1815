"""CPU-side checks of B200_expand_edges: argument, domain, dimension and index errors come back before any device work,
host-resident forward layers are refused, and without a GPU the call fails loudly before any host work (there is no CPU
fallback).  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Matrix, TensorLayers, TENSOR_LAYERS


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def call(src, types, ntypes=None, dir=fb.DIR_OUT, mode=fb.EDGES_ALL, targets=None, cap=16, p=True, nout=True):
    src = np.ascontiguousarray(src, dtype=np.uint64)
    ls = (TensorLayers * max(1, len(types or ())))()
    for k, t in enumerate(types or ()):
        for name in TENSOR_LAYERS:
            x = t.get(name)
            setattr(ls[k], name, None if x is None else x.h)
    tg = None if targets is None else np.ascontiguousarray(targets, dtype=np.uint64)
    pp = np.zeros(len(src) + 1, np.uint64)
    node, edge = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint64)
    nv = U64(0)
    return lib().B200_expand_edges(src.ctypes.data if len(src) else None, None if tg is None else tg.ctypes.data, len(src),
                                   None if types is None else ls, len(types or ()) if ntypes is None else ntypes, dir, mode,
                                   pp.ctypes.data if p else None, node.ctypes.data, edge.ctypes.data, None, None, cap,
                                   C.byref(nv) if nout else None)


def tensor(n=16, huge=False):
    nn = 1 << 60 if huge else n
    return {"m": Matrix(nn, nn, "u64"), "dp": Matrix(nn, nn, "u64"), "dm": Matrix(nn, nn), "mt": Matrix(nn, nn),
            "mt_dp": Matrix(nn, nn), "mt_dm": Matrix(nn, nn), "me": Matrix(1 << 60, 1 << 60), "me_dp": Matrix(1 << 60, 1 << 60),
            "me_dm": Matrix(1 << 60, 1 << 60)}


def test_null_pointers():
    fb.init()
    t = tensor()
    assert call([0], None, ntypes=1) == -2                                   # GrB_NULL_POINTER: types
    assert call([0], [t], p=False) == -2                                     # out_p
    assert call([0], [t], nout=False) == -2                                  # nout
    assert call([0], [dict(t, m=None)]) == -2                                # m
    for d in (fb.DIR_IN, fb.DIR_BOTH):
        assert call([0], [dict(t, mt=None)], dir=d) == -2                    # mt under IN / BOTH
    pp, nv = np.zeros(3, np.uint64), U64(0)
    ls = (TensorLayers * 1)()
    ls[0].m = t["m"].h
    assert lib().B200_expand_edges(None, None, 2, ls, 1, 0, 0, pp.ctypes.data, None, None, None, None, 0, C.byref(nv)) == -2
    assert lib().B200_expand_edges(np.zeros(1, np.uint64).ctypes.data, None, 1, ls, 1, 0, 0, pp.ctypes.data, None, None, None,
                                   None, 4, C.byref(nv)) == -2               # out_node / out_edge with a capacity


def test_values_domains_dimensions_indices():
    fb.init()
    t, small, rect = tensor(), tensor(8), Matrix(16, 8)
    assert call([0], [t], ntypes=0) == -3                                    # GrB_INVALID_VALUE: ntypes < 1
    assert call([0], [t], ntypes=65537) == -3                                # more types than out_type can name
    assert call([0], [t], dir=3) == -3 and call([0], [t], dir=-1) == -3      # dir out of range
    assert call([0], [t], mode=2) == -3 and call([0], [t], mode=-1) == -3    # mode out of range
    assert call([0], [dict(t, m=Matrix(16, 16))]) == -5                      # GrB_DOMAIN_MISMATCH: m not UINT64
    assert call([0], [dict(t, dp=Matrix(16, 16))]) == -5                     # dp not UINT64
    assert call([0], [dict(t, m=Matrix(16, 8, "u64"))]) == -6                # GrB_DIMENSION_MISMATCH: not square
    assert call([0], [t, small]) == -6                                       # types of different sizes
    for k in ("dp", "dm", "mt", "mt_dp", "mt_dm"):
        assert call([0], [dict(t, **{k: small[k]})]) == -6, k                # a layer not shaped like m
    assert call([0], [dict(t, mt=rect)], dir=fb.DIR_IN) == -6
    assert call([16], [t]) == -4                                             # GrB_INVALID_INDEX: a source >= n
    assert call([0, 3], [t], targets=[1, 16]) == -4                          # a target >= n


def test_host_resident_forward_layers_are_refused():
    assert call([0], [tensor(huge=True)]) == -8                              # GrB_NOT_IMPLEMENTED
    assert call([0], [tensor(huge=True)], dir=fb.DIR_BOTH) == -8


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_expand_edges_fails_loudly_without_gpu():
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes")
    for d in (fb.DIR_OUT, fb.DIR_IN, fb.DIR_BOTH):
        for mode in (fb.EDGES_ALL, fb.EDGES_FIRST):
            assert call([0, 1], [t, t], dir=d, mode=mode) == -7002           # GxB_GPU_ERROR
            assert call([0], [t], dir=d, mode=mode, targets=[1]) == -7002
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes")) == before
    assert t["m"].pending()                                                  # the queued write was not finished by the call
    with pytest.raises(fb.GrbError) as e:
        fb.expand_edges([0], [t], fb.DIR_OUT)
    assert e.value.info == -7002
