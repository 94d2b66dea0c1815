"""Hot-set-ordered frontiers (bits_hop.cu: permuted form): every observer of an ordered intermediate.  The 3-hop chain through this path
is also checked by bench.py's all-rows digest parity; this test adds the other observers.  Last in the `pytest -x` order."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200._lib import lib, obj, check, P, U64
from falkordb_b200.grb import Matrix, Descriptor
from test_gpu_parity import to_dev, assert_same, bitmap_of, diag_csr
from test_host_tensor import run as run_host_test

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("nsrc", [6, 64, 300])
def test_frontier_in_hot_set_order_between_push_and_pull(nsrc):
    """With the pull tables in place (B200_Matrix_prepare) a CSR frontier pushed through A lands in A's hot-set order and the next
    pull gathers from it directly.  Every way of looking at such an intermediate must see the natural-order content: nvals, wait
    + export, the bitmap hand-off, the row iterator, dup, use as a mask, union with another frontier, a hop through a DIFFERENT
    matrix, the push direction, a diagonal filter -- and the plain chain must match the oracle with the option on and off."""
    A = orc.rmat_csr(15, 16, 31)
    B = orc.rmat_csr(15, 8, 32)
    n = A.nrows
    rng = np.random.default_rng(nsrc)
    src = rng.choice(np.nonzero(np.diff(A.p))[0], size=nsrc, replace=False)
    dA, dB = to_dev(A).prepare(True), to_dev(B).prepare(True)
    F1 = orc.mxm(orc.build_matrix(nsrc, n, np.arange(nsrc), src), A)
    F2 = orc.mxm(F1, A)
    F3 = orc.mxm(F2, A)

    pushed = []

    def two_hops():
        fb.set_option("pull_mode", -1)  # a forced pull would bypass the CSR push
        F = Matrix(nsrc, n, bool)
        F.build(np.arange(nsrc), src)
        fb.set_option("bits_mode", 0)   # hop 1 row-wise (a CSR result), as the auto mode does for a one-entry-per-row frontier
        F.lmxm(dA)
        fb.set_option("bits_mode", 1)
        F.lmxm(dA)                      # CSR push while the expansion is small: the result is in dA's order when perm_push is on
        pushed.append(fb.get_stat("last_path") == 7)
        fb.set_option("pull_mode", 1)
        return F

    fb.set_option("bits_mode", 1)
    try:
        for perm in (1, 0):
            fb.set_option("perm_push", perm)
            F = two_hops()
            F.lmxm(dA)
            assert fb.get_stat("last_path") == 3
            assert_same(F, F3, f"3-hop chain, perm_push={perm}")
        fb.set_option("perm_push", 1)
        F = two_hops()
        assert F.nvals() == F2.nnz
        assert_same(F, F2, "intermediate observed through wait + export")
        F = two_hops()
        wpr = (n + 63) // 64
        bm = np.zeros((nsrc, wpr), np.uint64)
        F.export_bitmap(bm)
        assert np.array_equal(bm, bitmap_of(F2)), "bitmap hand-off of an intermediate"
        F = two_hops()
        D = F.dup()
        D.lmxm(dA)
        assert_same(D, F3, "dup of an ordered frontier, then the pull")
        assert_same(F, F2, "the original after its dup was multiplied")
        F = two_hops()
        F.lmxm(dB)                      # ordered for dA, multiplied by dB
        assert_same(F, orc.mxm(F2, B), "hop through a different matrix")
        F = two_hops()
        fb.set_option("pull_mode", 0)
        F.lmxm(dA)
        assert fb.get_stat("last_path") == 2
        assert_same(F, F3, "push direction from an ordered frontier")
        fb.set_option("pull_mode", 1)
        M = two_hops()                  # as the complemented mask of another product: C<!M, replace> = G * A
        G = Matrix(nsrc, n, bool)
        G.build(np.arange(nsrc), src)
        G.mxm(G, dA, M, Descriptor.RSC)
        assert_same(G, orc.mxm(orc.build_matrix(nsrc, n, np.arange(nsrc), src), A, F2, 2), "ordered frontier as a mask")
        U = two_hops()
        V = Matrix(nsrc, n, bool)
        V.build(np.arange(nsrc), src)
        V.lmxm(dB)
        U.element_wise_add(None, None, V, None)
        assert_same(U, orc.ewise_add(F2, orc.mxm(orc.build_matrix(nsrc, n, np.arange(nsrc), src), B)), "union with a natural-order frontier")
        lab = diag_csr(n, rng.choice(n, n // 2, replace=False))
        F = two_hops()
        F.lmxm(to_dev(lab))
        assert_same(F, orc.mxm(F2, lab), "diagonal filter after an ordered push")
        if nsrc <= 64:
            F = two_hops()
            wr = np.repeat(np.arange(nsrc), np.diff(F2.p))
            assert list(F.iter()) == list(zip(wr.tolist(), F2.j.tolist())), "row iterator over an ordered frontier"
        # the CSR push takes a hop iff its expansion is small against A (flops * 4 <= nnz(A), csr_push.cu: bits_push_from_csr)
        expect_push = int(np.diff(A.p)[F1.j].sum()) * 4 <= A.nnz
        assert all(p == expect_push for p in pushed), (expect_push, pushed)
        if nsrc <= 6:
            assert expect_push, "the small case is meant to exercise the ordered form"
    finally:
        for k, v in (("bits_mode", -1), ("pull_mode", -1), ("perm_push", 1)):
            fb.set_option(k, v)
