"""Dirty hops in one pass: B200_Matrix_delta_lmxm (F <- (F*m AND NOT F*dm) OR F*dp with the delta terms applied in place) and
B200_traverse_batch_delta, against the oracle's delta_lmxm and against the reference's three-mxm composition
(Matrix.delta_lmxm), bit for bit and flop for flop."""
import ctypes as C
import os

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def host():
    L = C.CDLL(os.path.join(ROOT, "falkordb_b200", "libfdbhost.so"))
    L.fdbh_run_test.argtypes = [C.c_char_p]
    L.fdbh_last_message.restype = C.c_char_p
    L.fdbh_vm_from_csr.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
    L.fdbh_vm_from_csr.restype = C.c_void_p
    L.fdbh_vm_free.argtypes = [C.c_void_p]
    L.fdbh_vm_set.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    L.fdbh_vm_remove.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64]
    args = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64,
            C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    L.fdbh_expand_batch.argtypes = args
    L.fdbh_expand_batch_fused.argtypes = args
    L.fdbh_expand_batch_coalesced.argtypes = args + [C.c_int]
    L.fdbh_free.argtypes = [C.c_void_p]
    return L


def vm_from(L, c):
    p = c.p.astype(np.uint64)
    h = L.fdbh_vm_from_csr(c.nrows, c.ncols, p.ctypes.data, c.j.ctypes.data if c.nnz else None)
    assert h, L.fdbh_last_message().decode()
    return h


def expand(L, src, hops, sl=(), dl=(), fused=False, coalesced=False):
    """(row, dest) pairs of the host CondTraverse mirror: per-hop delta_lmxm, or every hop in one call (coalesced)"""
    src = np.ascontiguousarray(src, dtype=np.uint64)
    arr = lambda hs: (C.c_void_p * max(1, len(hs)))(*hs)
    rows, dest, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
    args = (src.ctypes.data, len(src), arr(hops), len(hops), arr(sl), len(sl), arr(dl), len(dl), C.byref(rows), C.byref(dest),
            C.byref(n))
    if coalesced:
        rc = L.fdbh_expand_batch_coalesced(*args, int(fused))
    else:
        rc = (L.fdbh_expand_batch_fused if fused else L.fdbh_expand_batch)(*args)
    assert rc == 0, L.fdbh_last_message().decode()
    r = np.ctypeslib.as_array(C.cast(rows, C.POINTER(C.c_uint64)), shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
    d = np.ctypeslib.as_array(C.cast(dest, C.POINTER(C.c_uint64)), shape=(n.value,)).copy() if n.value else np.zeros(0, np.uint64)
    L.fdbh_free(rows); L.fdbh_free(dest)
    return r, d


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    yield
    for k, v in (("bits_mode", -1), ("pull_mode", -1), ("csr_push", 1), ("diag_filter", 1)):
        fb.set_option(k, v)


def to_dev(c, dtype=bool):
    x = None
    if dtype == "u64":
        x = np.arange(1, c.nnz + 1, dtype=np.uint64) if c.x is None else c.x
    return Matrix.import_csr(c.nrows, c.ncols, c.p.astype(np.uint64), c.j, x, dtype)


def from_dev(m):
    p, j, _ = m.export_csr()
    return orc.CSR(m.nrows(), m.ncols(), p, j, None)


def same(dev, want, what):
    got = from_dev(dev)
    assert np.array_equal(got.p, want.p) and np.array_equal(got.j, want.j), what


def graph(scale=12, seed=3):
    A = orc.rmat_csr(scale, 8, seed)
    return A, to_dev(A).prepare()


def deltas(rng, A, ndel, nadd, overlap=0, outside=0):
    """dm: ndel entries of A plus `outside` pairs that are not in A; dp: nadd new pairs plus `overlap` entries already in A."""
    n = A.nrows
    rows, cols, _ = A.tuples()
    have = A.tuple_set()
    take = rng.choice(A.nnz, ndel + overlap, replace=False)
    fresh = lambda k: [t for t in zip(rng.integers(0, n, 4 * k + 8).tolist(), rng.integers(0, n, 4 * k + 8).tolist())
                       if t not in have][:k]
    out = fresh(outside)
    dm = orc.build_matrix(n, n, np.r_[rows[take[:ndel]], [a for a, _ in out]], np.r_[cols[take[:ndel]], [b for _, b in out]])
    add = fresh(nadd)
    dp = orc.build_matrix(n, n, np.r_[[a for a, _ in add], rows[take[ndel:]]], np.r_[[b for _, b in add], cols[take[ndel:]]])
    return dp, dm


def sources(rng, A, nsrc):
    """nsrc distinct sources, the first of them isolated (no out-edges) when the graph has one."""
    iso = np.nonzero(np.diff(A.p) == 0)[0]
    live = np.nonzero(np.diff(A.p))[0]
    src = rng.choice(live, nsrc, replace=False)
    if len(iso):
        src[0] = iso[0]
    return src


def frontier(A, src):
    F = Matrix(len(src), A.nrows, bool)
    F.build(np.arange(len(src)), src)
    return F


def run_both(F1, F2, m, dp, dm):
    """F1 by the composition, F2 by the fused entry; returns (composition flops, fused flops, fused path)."""
    fb.reset_stats()
    F1.delta_lmxm(m, dp, dm)
    fc = fb.get_stat("total_flops")
    fb.reset_stats()
    F2.delta_lmxm_fused(m, dp, dm)
    return fc, fb.get_stat("total_flops"), fb.get_stat("last_path")


@pytest.mark.parametrize("nsrc", [1, 100, 250, 500, 1000])          # W = 1, 2, 4, 8, 16
@pytest.mark.parametrize("pull_mode", [-1, 0, 1])
@pytest.mark.parametrize("bits_mode", [1, 0])
def test_delta_lmxm_two_hops_match_oracle_and_composition(nsrc, pull_mode, bits_mode):
    rng = np.random.default_rng(nsrc + 7 * (pull_mode + 1))
    A, Ad = graph()
    dp, dm = deltas(rng, A, 300, 300, overlap=20, outside=20)
    dpd, dmd = to_dev(dp), to_dev(dm)
    src = sources(rng, A, nsrc)
    fb.set_option("bits_mode", bits_mode)
    fb.set_option("pull_mode", pull_mode)
    F1, F2 = frontier(A, src), frontier(A, src)
    W = orc.build_matrix(nsrc, A.nrows, np.arange(nsrc), src)
    for hop in range(2):                                     # hop 1 from the CSR frontier, hop 2 from the bit-matrix
        W = orc.delta_lmxm(W, A, dp, dm)
        fc, ff, path = run_both(F1, F2, Ad, dpd, dmd)
        assert ff == fc, f"hop {hop}: flops {ff} != composition's {fc}"
        if bits_mode == 0:
            assert path in (1, 6)
        same(F2, W, f"hop {hop}: fused vs oracle")
        same(F1, W, f"hop {hop}: composition vs oracle")


def test_ordered_frontier_survives_a_dirty_hop():
    """push (CSR frontier -> hot-set order of m) then pull straight from that order, both hops dirty"""
    rng = np.random.default_rng(11)
    A, Ad = graph(13, 5)
    dp, dm = deltas(rng, A, 2000, 2000, overlap=50, outside=50)
    dpd, dmd = to_dev(dp), to_dev(dm)
    src = sources(rng, A, 300)
    fb.set_option("bits_mode", 1)
    F1, F2 = frontier(A, src), frontier(A, src)
    W = orc.build_matrix(len(src), A.nrows, np.arange(len(src)), src)
    for hop, pm in enumerate((-1, 1)):
        fb.set_option("pull_mode", pm)
        W = orc.delta_lmxm(W, A, dp, dm)
        fc, ff, path = run_both(F1, F2, Ad, dpd, dmd)
        assert path == (7, 3)[hop], f"hop {hop} took path {path}"
        assert ff == fc
        same(F2, W, f"hop {hop}")
        same(F1, W, f"hop {hop} composition")


def test_diagonal_label_operand_with_dirty_deltas():
    rng = np.random.default_rng(5)
    A, Ad = graph()
    n = A.nrows
    lab = np.sort(rng.choice(n, n // 3, replace=False))
    L = orc.build_matrix(n, n, lab, lab)
    drop = rng.choice(lab, 60, replace=False)
    add = np.setdiff1d(rng.choice(n, 120, replace=False), lab)
    dm, dp = orc.build_matrix(n, n, drop, drop), orc.build_matrix(n, n, add, add)
    Ld, dpd, dmd = to_dev(L), to_dev(dp), to_dev(dm)
    src = sources(rng, A, 200)
    for bits_mode in (1, 0):
        fb.set_option("bits_mode", bits_mode)
        F1, F2 = frontier(A, src), frontier(A, src)
        W = orc.build_matrix(len(src), n, np.arange(len(src)), src)
        for M, Md, dd in ((A, Ad, None), (L, Ld, (dpd, dmd))):
            W = orc.delta_lmxm(W, M, dp, dm) if dd else orc.mxm(W, M)
            if dd:
                fc, ff, path = run_both(F1, F2, Md, *dd)
                assert ff == fc
                if bits_mode == 1:
                    assert path == 5
            else:
                F1.lmxm(Md)
                F2.lmxm(Md)
        same(F2, W, f"label hop, bits_mode {bits_mode}")
        same(F1, W, f"label hop composition, bits_mode {bits_mode}")


def test_uint64_tensor_operands_and_pending_deltas():
    rng = np.random.default_rng(9)
    A, _ = graph()
    dp, dm = deltas(rng, A, 200, 200)
    m = to_dev(A, "u64").prepare()
    dpd = to_dev(dp, "u64")
    dmd = Matrix(A.nrows, A.ncols, bool)                     # dm with pending tuples: finished first, as dm.wait() does
    r, c, _ = dm.tuples()
    for a, b in zip(r, c):
        dmd.set(int(a), int(b))
    assert dmd.pending()
    src = sources(rng, A, 400)
    for bits_mode in (1, -1):
        fb.set_option("bits_mode", bits_mode)
        F1, F2 = frontier(A, src), frontier(A, src)
        W = orc.build_matrix(len(src), A.nrows, np.arange(len(src)), src)
        for _ in range(3):
            W = orc.delta_lmxm(W, A, dp, dm)
            fc, ff, _ = run_both(F1, F2, m, dpd, dmd)
            assert ff == fc
            same(F2, W, f"u64 operands, bits_mode {bits_mode}")


@pytest.mark.parametrize("which", ["none", "empty", "dp_only", "dm_only"])
def test_null_and_empty_deltas(which):
    rng = np.random.default_rng(2)
    A, Ad = graph()
    n = A.nrows
    dp, dm = deltas(rng, A, 100, 100)
    E = orc.build_matrix(n, n, [], [])
    pick = {"none": (None, None), "empty": (E, E), "dp_only": (dp, None), "dm_only": (None, dm)}[which]
    dev = [None if x is None else to_dev(x) for x in pick]
    src = sources(rng, A, 64)
    fb.set_option("bits_mode", 1)
    F = frontier(A, src)
    W = orc.build_matrix(len(src), n, np.arange(len(src)), src)
    for _ in range(2):
        W = orc.delta_lmxm(W, A, pick[0] if pick[0] is not None else E, pick[1] if pick[1] is not None else E)
        F.delta_lmxm_fused(Ad, *dev)
        same(F, W, which)


def test_bad_arguments():
    A, Ad = graph(8, 1)
    F = Matrix(4, A.nrows, bool)
    small = Matrix(8, 8, bool)
    with pytest.raises(fb.GrbError) as e:
        F.delta_lmxm_fused(Ad, small, None)
    assert e.value.info == -6
    with pytest.raises(fb.GrbError) as e:
        Matrix(4, 8, bool).delta_lmxm_fused(Ad, None, None)
    assert e.value.info == -6


def chain_oracle(A, src, hop_deltas):
    W = orc.build_matrix(len(src), A.nrows, np.arange(len(src)), src)
    E = orc.build_matrix(A.nrows, A.ncols, [], [])
    for d in hop_deltas:
        W = orc.delta_lmxm(W, A, d[0] if d and d[0] is not None else E, d[1] if d and d[1] is not None else E)
    return W


@pytest.mark.parametrize("nsrc", [3, 300, 1000])
def test_traverse_batch_delta_formats(nsrc):
    rng = np.random.default_rng(nsrc)
    A, Ad = graph()
    n = A.nrows
    dp, dm = deltas(rng, A, 400, 400, overlap=10, outside=10)
    dpd, dmd = to_dev(dp), to_dev(dm)
    hop_deltas = [(dp, dm), None, (None, dm)]
    devd = [(dpd, dmd), (None, None), (None, dmd)]
    src = sources(rng, A, nsrc)
    want = chain_oracle(A, src, hop_deltas)
    wpr = (n + 63) // 64
    fb.set_option("bits_mode", 1)
    p_ = np.zeros(nsrc + 1, np.uint64)
    j_ = np.zeros(max(1, want.nnz), np.uint32)
    fl, nv, fmt = fb.traverse_batch(src, [Ad] * 3, fb.OUT_CSR, out_p=p_, out_j=j_, deltas=devd)
    assert fmt == fb.OUT_CSR and nv == want.nnz
    assert np.array_equal(p_.astype(np.int64), want.p) and np.array_equal(j_[:want.nnz], want.j)
    bm = np.zeros((nsrc, wpr), np.uint64)
    fl2, nv2, fmt = fb.traverse_batch(src, [Ad] * 3, fb.OUT_BITMAP, out_bitmap=bm, deltas=devd)
    assert fmt == fb.OUT_BITMAP and fl2 == fl
    wbm = np.zeros((nsrc, wpr), np.uint64)
    rows, cols, _ = want.tuples()
    np.bitwise_or.at(wbm, (rows.astype(np.int64), (cols // 64).astype(np.int64)), np.left_shift(np.uint64(1), (cols % 64).astype(np.uint64)))
    assert np.array_equal(bm, wbm)
    bm[:] = 0
    fl3, nv3, fmt = fb.traverse_batch(src, [Ad] * 3, fb.OUT_AUTO, out_bitmap=bm, out_p=p_, out_j=j_, deltas=devd)
    assert fl3 == fl and nv3 == want.nnz
    if fmt == fb.OUT_BITMAP:
        assert np.array_equal(bm, wbm)
    else:
        assert np.array_equal(p_.astype(np.int64), want.p) and np.array_equal(j_[:want.nnz], want.j)
    # the composition's flops: one delta_lmxm per hop through Matrix.delta_lmxm
    F = frontier(A, src)
    E = Matrix(n, n, bool)
    fb.reset_stats()
    for d in devd:
        F.delta_lmxm(Ad, d[0] or E, d[1] or E)
    assert fb.get_stat("total_flops") == fl
    if want.nnz:
        with pytest.raises(BufferError):
            fb.traverse_batch(src, [Ad] * 3, fb.OUT_CSR, out_p=p_, out_j=j_[: want.nnz - 1], deltas=devd)
    # no deltas at all: the clean traversal
    clean = chain_oracle(A, src, [None] * 3)
    fl0, nv0, _ = fb.traverse_batch(src, [Ad] * 3, fb.OUT_CSR, out_p=p_, out_j=np.zeros(max(1, clean.nnz), np.uint32),
                                    deltas=[(None, None)] * 3)
    assert nv0 == clean.nnz and np.array_equal(p_.astype(np.int64), clean.p)


def test_traverse_batch_delta_rejects_mismatched_deltas():
    A, Ad = graph(8, 1)
    small = Matrix(8, 8, bool)
    p_ = np.zeros(3, np.uint64)
    with pytest.raises(fb.GrbError) as e:
        fb.traverse_batch([0, 1], [Ad], fb.OUT_CSR, out_p=p_, out_j=np.zeros(16, np.uint32), deltas=[(small, None)])
    assert e.value.info == -6


def test_host_coalesced_expand_matches_per_hop_expand():
    """the dirty-snapshot and dirty-label cases of the per-hop host traversal, clean and dirty VersionedMatrix hops"""
    L = host()
    A = orc.rmat_csr(11, 8, 9)
    n = A.nrows
    rng = np.random.default_rng(2)
    src = rng.choice(np.nonzero(np.diff(A.p))[0], 200, replace=False)
    vA, vB = vm_from(L, A), vm_from(L, A)
    rows, cols, _ = A.tuples()
    for q in rng.choice(A.nnz, 300, replace=False):
        assert L.fdbh_vm_remove(vB, int(rows[q]), int(cols[q])) == 0
    have = A.tuple_set()
    for a, b in sorted({(int(a), int(b)) for a, b in zip(rng.integers(0, n, 300), rng.integers(0, n, 300))} - have):
        assert L.fdbh_vm_set(vB, a, b) == 0
    lab_s = np.sort(rng.choice(n, n // 2, replace=False))
    lab_d = np.sort(rng.choice(n, n // 3, replace=False))
    vs = vm_from(L, orc.build_matrix(n, n, lab_s, lab_s))
    vd = vm_from(L, orc.build_matrix(n, n, lab_d, lab_d))
    for v in rng.choice(lab_d, 50, replace=False):
        assert L.fdbh_vm_remove(vd, int(v), int(v)) == 0
    for v in np.setdiff1d(rng.choice(n, 100, replace=False), lab_d):
        assert L.fdbh_vm_set(vd, int(v), int(v)) == 0
    cases = [([vA, vA, vA], [], []), ([vB], [], []), ([vB, vA, vB], [vs], [vd]), ([vA, vA], [], [vd])]
    for hops, sl, dl in cases:
        for fuse in (False, True):
            r0, d0 = expand(L, src, hops, sl, dl, fused=fuse)
            r1, d1 = expand(L, src, hops, sl, dl, fused=fuse, coalesced=True)
            assert np.array_equal(r0, r1) and np.array_equal(d0, d1), (len(hops), len(sl), len(dl), fuse)
    for h in (vA, vB, vs, vd):
        L.fdbh_vm_free(h)
    assert L.fdbh_run_test(b"coalesced_traverse_over_tensor_operand") == 0, L.fdbh_last_message().decode()
