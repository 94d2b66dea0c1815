"""Full size: the adjacency of algo.WCC / algo.labelPropagation over RMAT-24 (edge factor 16, seed 1) split into 3 relationship types
by an edge hash, each with |dp| = |dm| = 10^5 pending.  B200_adjacency_delta's symmetric output must equal, by digest, the reference's
route composed from the library's own set operations ((m \\ dm) u dp per type, their union, its transpose and one more union); its
kept-list output (1 % of the vertices) the same union's induced subgraph computed on the host; and LAGr_ConnectedComponents must give
the same components on both symmetric matrices."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200._lib import lib, check, P
from falkordb_b200.grb import Descriptor, Matrix
from fullsize_util import need, rmat_both, defaults, same_digest

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def components(A, n):
    """LAGr_ConnectedComponents on a symmetric matrix (the graph takes a duplicate)"""
    L = lib()
    G, h = P(), P()
    check(L.GrB_Matrix_dup(C.byref(h), A.h))
    assert L.LAGraph_New(C.byref(G), C.byref(h), 0, None) == 0              # LAGraph_ADJACENCY_UNDIRECTED
    comp = P()
    info = L.LAGr_ConnectedComponents(C.byref(comp), G, None)
    L.LAGraph_Delete(C.byref(G), None)
    assert info == 0
    nv = C.c_uint64(n)
    I, X = np.empty(n, np.uint64), np.empty(n, np.int64)
    check(L.GrB_Vector_extractTuples_INT64(I.ctypes.data, X.ctypes.data, C.byref(nv), comp))
    L.GrB_Vector_free(C.byref(comp))
    assert nv.value == n
    return X


def test_adjacency_rmat24_three_types_equals_the_reference_route():
    need(30, 24)          # device: the types, their deltas, two symmetric unions; host: the exported union and its split
    scale, ntypes, ndelta = 24, 3, 100_000
    n = 1 << scale
    _, Ao = rmat_both(scale, 1)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(Ao.p))
    cols = Ao.j.astype(np.uint64)
    kind = (((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F))) >> np.uint64(61)) % np.uint64(ntypes)
    rng = np.random.default_rng(6)
    ops = []
    for t in range(ntypes):
        sel = np.nonzero(kind == t)[0]
        pt = np.zeros(n + 1, np.uint64)
        np.cumsum(np.bincount(rows[sel].astype(np.int64), minlength=n), out=pt[1:])
        m = Matrix.import_csr(n, n, pt, Ao.j[sel], None, bool)
        pick = rng.choice(len(sel), ndelta, replace=False)
        dm, dp = Matrix(n, n, bool), Matrix(n, n, bool)
        dm.build(rows[sel][pick], cols[sel][pick])
        dp.build(rng.integers(0, n, ndelta).astype(np.uint64), rng.integers(0, n, ndelta).astype(np.uint64))
        ops.append((m, dp, dm))
    del rows, cols, kind
    U = Matrix(n, n, bool)
    for m, dp, dm in ops:                       # U |= (m \ dm) u dp, through the library's own set operations
        E = Matrix(n, n, bool)
        E.element_wise_add(dm, m, m, Descriptor.RC)
        E.element_wise_add(None, E, dp)
        U.element_wise_add(None, U, E)
        del E
    U.wait()
    S = Matrix(n, n, bool)                      # build_symmetric_adjacency_matrix: U + U'
    S.element_wise_add(None, U, U.transpose())
    S.wait()
    ms, deltas = [o[0] for o in ops], [(o[1], o[2]) for o in ops]

    A = fb.adjacency(ms, deltas=deltas, symmetric=True)
    same_digest(A, S.digest(), "symmetric adjacency")
    assert np.array_equal(components(A, n), components(S, n)), "WCC differs from the reference route's"
    del A, S

    keep = np.sort(rng.choice(n, n // 100, replace=False)).astype(np.uint64)
    K = fb.adjacency(ms, deltas=deltas, keep=keep)
    p, j, _ = U.export_csr()
    del U
    rank = np.full(n, -1, np.int64)
    rank[keep.astype(np.int64)] = np.arange(len(keep))
    r = rank[np.repeat(np.arange(n, dtype=np.int64), np.diff(p))]
    c = rank[j.astype(np.int64)]
    inside = (r >= 0) & (c >= 0)
    want = orc.build_matrix(len(keep), len(keep), r[inside], c[inside])
    del p, j, r, c, inside
    assert want.nnz > 1000
    same_digest(K, orc.digest(want), "kept-list adjacency")
