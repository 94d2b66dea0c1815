"""CPU-side checks of B200_Tensor_insert_plan / B200_Tensor_remove_plan: argument, domain, dimension and index errors come back
before any device work, host-resident forward layers are refused, an empty batch succeeds with no device work, and without a GPU
the calls fail loudly before any host work (there is no CPU fallback).  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Matrix, TensorLayers, TENSOR_LAYERS


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def tensor(n=16, huge=False):
    nn = 1 << 60 if huge else n
    return {"m": Matrix(nn, nn, "u64"), "dp": Matrix(nn, nn, "u64"), "dm": Matrix(nn, nn), "mt": Matrix(nn, nn),
            "mt_dp": Matrix(nn, nn), "mt_dm": Matrix(nn, nn), "me": Matrix(1 << 60, 1 << 60), "me_dp": Matrix(1 << 60, 1 << 60),
            "me_dm": Matrix(1 << 60, 1 << 60)}


def call(fn, t, a, b, c, outs=True, counts=True, layers=True):
    """fn = 'insert' (a, b, c = srcs, dsts, ids) or 'remove' (ids, srcs, dsts)"""
    a, b, c = (np.ascontiguousarray(x, dtype=np.uint64) for x in (a, b, c))
    n = len(a)
    ls = TensorLayers()
    for name in TENSOR_LAYERS:
        x = t.get(name)
        setattr(ls, name, None if x is None else x.h)
    r = [np.zeros(max(n, 1), np.uint64) for _ in range(3)] + [np.zeros(max(n, 1), np.uint8)]
    m = [np.zeros(max(2 * n, 1), np.uint64) for _ in range(2)] + [np.zeros(max(2 * n, 1), np.uint8)]
    nr, nm = U64(7), U64(7)
    f = lib().B200_Tensor_insert_plan if fn == "insert" else lib().B200_Tensor_remove_plan
    ptr = lambda x: x.ctypes.data if outs else None
    return f(C.byref(ls) if layers else None, a.ctypes.data if n else None, b.ctypes.data if n else None,
             c.ctypes.data if n else None, n, *[ptr(x) for x in r], C.byref(nr) if counts else None, *[ptr(x) for x in m],
             C.byref(nm) if counts else None)


FNS = ("insert", "remove")


@pytest.mark.parametrize("fn", FNS)
def test_null_pointers(fn):
    fb.init()
    t = tensor()
    assert call(fn, t, [0], [1], [2], layers=False) == -2                # GrB_NULL_POINTER: the layers
    assert call(fn, dict(t, m=None), [0], [1], [2]) == -2                 # m
    assert call(fn, dict(t, mt=None), [0], [1], [2]) == -2                # mt
    assert call(fn, t, [0], [1], [2], counts=False) == -2                 # nin / nme
    assert call(fn, t, [0], [1], [2], outs=False) == -2                   # output arrays with a batch
    assert call(fn, t, [], [], [], counts=False) == -2                    # the counts even for an empty batch


@pytest.mark.parametrize("fn", FNS)
def test_domains_dimensions_indices(fn):
    fb.init()
    t, small = tensor(), tensor(8)
    ok = ([0], [1], [2]) if fn == "insert" else ([2], [0], [1])
    assert call(fn, dict(t, m=Matrix(16, 16)), *ok) == -5                 # GrB_DOMAIN_MISMATCH: m not UINT64
    assert call(fn, dict(t, dp=Matrix(16, 16)), *ok) == -5                # dp not UINT64
    assert call(fn, dict(t, m=Matrix(16, 8, "u64")), *ok) == -6           # GrB_DIMENSION_MISMATCH: not square
    for k in ("dp", "dm", "mt", "mt_dp", "mt_dm"):
        assert call(fn, dict(t, **{k: small[k]}), *ok) == -6, k           # a layer not shaped like m
    big = 1 << 60
    if fn == "insert":
        bad = (([16], [1], [2]), ([0], [16], [2]), ([0], [1], [big]), ([0, 0], [1, 1], [2, big]))
    else:
        bad = (([2], [16], [1]), ([2], [0], [16]), ([big], [0], [1]), ([2, big], [0, 0], [1, 1]))
    for args in bad:
        assert call(fn, t, *args) == -4, args                             # GrB_INVALID_INDEX: vertex >= n or id >= 2^60


@pytest.mark.parametrize("fn", FNS)
def test_host_resident_forward_layers_are_refused(fn):
    assert call(fn, tensor(huge=True), [0], [1], [2]) == -8              # GrB_NOT_IMPLEMENTED


@pytest.mark.parametrize("fn", FNS)
def test_empty_batch_is_success_with_no_device_work(fn):
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    assert call(fn, t, [], [], []) == 0
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before
    assert t["m"].pending()                                               # nothing was finished either
    p = fb.insert_plan(t, [], [], []) if fn == "insert" else fb.remove_plan(t, [], [], [])
    assert all(len(v) == 0 for v in p.values())


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
@pytest.mark.parametrize("fn", FNS)
def test_plans_fail_loudly_without_gpu(fn):
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    t["dp"].set(2, 3, 9)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes")
    assert call(fn, t, [0, 2], [1, 3], [4, 5]) == -7002                   # GxB_GPU_ERROR
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes")) == before
    assert t["m"].pending() and t["dp"].pending()                        # the queued writes were not finished by the call
    with pytest.raises(fb.GrbError) as e:
        if fn == "insert":
            fb.insert_plan(t, [0], [1], [4])
        else:
            fb.remove_plan(t, [4], [0], [1])
    assert e.value.info == -7002


def test_symbols_resolve():
    for name in ("B200_Tensor_insert_plan", "B200_Tensor_remove_plan"):
        assert getattr(lib(), name) is not None
    from falkordb_b200 import host_mirror as hm
    L = hm.host()
    for name in ("fdbh_tensor_set_all_dev", "fdbh_tensor_remove_all_dev", "fdbh_tensor_remove_all_emptied", "fdbh_tensor_counts",
                 "fdbh_tensor_dup", "fdbh_tensor_fold_oversized", "fdbh_tensor_flush", "fdbh_tensor_edge_count", "fdbh_vm_set_all",
                 "fdbh_vm_state", "fdbh_run_write_test"):
        assert getattr(L, name) is not None, name
    assert hm.WRITE_REFERENCE == 0 and hm.WRITE_DEVICE == 1
    assert (fb.grb.PLAN_COMMITTED, fb.grb.PLAN_CANCEL, fb.grb.PLAN_MT_BASE, fb.grb.PLAN_EMPTIED, fb.grb.PLAN_DEMOTED,
            fb.grb.PLAN_M_HAS, fb.grb.PLAN_M_EQ) == (1, 2, 4, 8, 16, 32, 64)
