"""CPU-side checks of B200_var_len_trails: argument, domain, dimension and index errors come back before any device work, empty
batches and empty hop windows succeed with no device work, and without a GPU the call fails loudly before any host work (there is
no CPU fallback).  No kernel is launched here."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, P, U64
from falkordb_b200.grb import Matrix, TensorLayers, TENSOR_LAYERS

U64MAX = (1 << 64) - 1


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def call(starts, types, ntypes=None, dir=fb.DIR_OUT, lo=1, hi=3, dests=None, labels=(), nlabels=None, cap=16, pcap=16,
         p=True, nout=True, npath=True, end=True, hops=True, pe=True, pn=True):
    starts = np.ascontiguousarray(starts, dtype=np.uint64)
    ls = (TensorLayers * max(1, len(types or ())))()
    for k, t in enumerate(types or ()):
        for name in TENSOR_LAYERS:
            x = t.get(name)
            setattr(ls[k], name, None if x is None else x.h)
    nl = len(labels)
    lm, ldp, ldm = (P * max(1, nl))(), (P * max(1, nl))(), (P * max(1, nl))()
    for k, lab in enumerate(labels):
        if lab is not None:
            lm[k], ldp[k], ldm[k] = (None if x is None else x.h for x in lab)
    ds = None if dests is None else np.ascontiguousarray(dests, dtype=np.int64)
    pp = np.zeros(len(starts) + 1, np.uint64)
    oe, oh = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint32)
    ope, opn = np.zeros(max(pcap, 1), np.uint64), np.zeros(max(pcap + cap, 1), np.uint32)
    nv, npth = U64(7), U64(7)
    info = lib().B200_var_len_trails(starts.ctypes.data if len(starts) else None, None if ds is None else ds.ctypes.data, len(starts),
                                     None if types is None else ls, len(types or ()) if ntypes is None else ntypes, dir, lo, hi,
                                     lm, ldp, ldm, nl if nlabels is None else nlabels, U64MAX, pp.ctypes.data if p else None,
                                     oe.ctypes.data if end else None, oh.ctypes.data if hops else None, cap,
                                     ope.ctypes.data if pe else None, opn.ctypes.data if pn else None, pcap,
                                     C.byref(nv) if nout else None, C.byref(npth) if npath else None)
    return info, pp, nv.value, npth.value


def tensor(n=16, huge=False):
    nn = 1 << 60 if huge else n
    return {"m": Matrix(nn, nn, "u64"), "dp": Matrix(nn, nn, "u64"), "dm": Matrix(nn, nn), "mt": Matrix(nn, nn),
            "mt_dp": Matrix(nn, nn), "mt_dm": Matrix(nn, nn), "me": Matrix(1 << 60, 1 << 60), "me_dp": Matrix(1 << 60, 1 << 60),
            "me_dm": Matrix(1 << 60, 1 << 60)}


def label(n=16):
    return (Matrix(n, n), Matrix(n, n), Matrix(n, n))


def test_null_pointers():
    fb.init()
    t = tensor()
    assert call([0], None, ntypes=1)[0] == -2                               # GrB_NULL_POINTER: types
    assert call([0], [t], p=False)[0] == -2                                 # out_p
    assert call([0], [t], nout=False)[0] == -2                              # nout
    assert call([0], [t], npath=False)[0] == -2                             # npath
    assert call([0], [dict(t, m=None)])[0] == -2                            # m
    for d in (fb.DIR_IN, fb.DIR_BOTH):
        assert call([0], [dict(t, mt=None)], dir=d)[0] == -2                # mt under IN / BOTH
    assert call([0], [t], hops=False)[0] == -2                              # out_end without out_hops
    assert call([0], [t], pn=False)[0] == -2                                # path_edge without path_node
    pp, nv, npth = np.zeros(3, np.uint64), U64(0), U64(0)
    ls = (TensorLayers * 1)()
    ls[0].m = t["m"].h
    assert lib().B200_var_len_trails(None, None, 2, ls, 1, 0, 1, 2, None, None, None, 0, U64MAX, pp.ctypes.data, None, None, 0,
                                     None, None, 0, C.byref(nv), C.byref(npth)) == -2                  # starts
    assert lib().B200_var_len_trails(np.zeros(1, np.uint64).ctypes.data, None, 1, ls, 1, 0, 1, 2, None, None, None, 1, U64MAX,
                                     pp.ctypes.data, None, None, 0, None, None, 0, C.byref(nv), C.byref(npth)) == -2  # lab_m


def test_values_domains_dimensions_indices():
    fb.init()
    t, small = tensor(), tensor(8)
    assert call([0], [t], ntypes=0)[0] == -3                                # GrB_INVALID_VALUE: ntypes < 1
    assert call([0], [t], ntypes=65537)[0] == -3
    assert call([0], [t], dir=3)[0] == -3 and call([0], [t], dir=-1)[0] == -3
    assert call([0], [t], nlabels=-1)[0] == -3
    assert call([0], [dict(t, m=Matrix(16, 16))])[0] == -5                  # GrB_DOMAIN_MISMATCH: m not UINT64
    assert call([0], [dict(t, dp=Matrix(16, 16))])[0] == -5                 # dp not UINT64
    assert call([0], [dict(t, m=Matrix(16, 8, "u64"))])[0] == -6            # GrB_DIMENSION_MISMATCH
    assert call([0], [t, small])[0] == -6
    for k in ("dp", "dm", "mt", "mt_dp", "mt_dm"):
        assert call([0], [dict(t, **{k: small[k]})])[0] == -6, k
    for k in range(3):
        lab = list(label())
        lab[k] = Matrix(8, 8)
        assert call([0], [t], labels=[tuple(lab)])[0] == -6, k             # a label layer not n x n
    assert call([16], [t])[0] == -4                                         # GrB_INVALID_INDEX: a start >= n
    assert call([0, 3], [t], dests=[1, 16])[0] == -4                        # a destination >= n
    assert call([0], [tensor(huge=True)])[0] == -8                          # GrB_NOT_IMPLEMENTED: host-resident layers
    assert call([0], [t], labels=[label(1 << 40)])[0] in (-6, -8)           # a label of another size is refused first


def test_empty_batches_and_windows_do_no_device_work():
    fb.init()
    t = tensor()
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    info, pp, nv, npth = call([], [t])
    assert info == 0 and list(pp) == [0] and nv == 0 and npth == 0
    info, pp, nv, npth = call([0, 5, 5], [t], lo=3, hi=2)                   # min_hops > max_hops
    assert info == 0 and list(pp) == [0, 0, 0, 0] and nv == 0 and npth == 0
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_var_len_trails_fails_loudly_without_gpu():
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    for d in (fb.DIR_OUT, fb.DIR_IN, fb.DIR_BOTH):
        assert call([0, 1], [t, t], dir=d)[0] == -7002                      # GxB_GPU_ERROR
        assert call([0], [t], dir=d, lo=0, hi=U64MAX, dests=[1], labels=[label()])[0] == -7002
        assert call([0], [t], dir=d, labels=[None])[0] == -7002             # a missing label still needs the device
        assert call([0], [t], dir=d, end=False, hops=False, pe=False, pn=False)[0] == -7002   # count only
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before
    assert t["m"].pending()                                                 # the queued write was not finished by the call
    with pytest.raises(fb.GrbError) as e:
        fb.var_len_trails([0], [t])
    assert e.value.info == -7002
