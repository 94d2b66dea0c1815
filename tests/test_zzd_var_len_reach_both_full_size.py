"""Full size: B200_var_len_reach_both on a self-loop-free RMAT-16 tensor built on the device with pending writes (deletes, re-adds,
new pairs, new ids on loaded pairs), 512 starts, k = 3 and 4, checked without the DFS.  With M the effective multiplicity matrix
(test_zzc's `effective`) and P = pattern(M + M^T):
  rows, v != s   dist_P(s, v) <= k, by scipy level sweeps;
  the diagonal   g(s) <= k for the shortest cycle through s, computed independently of the device's bit split: g = 2 when
                 M[s, c] + M[c, s] >= 2 for some c, else the BFS tree from s with each vertex labelled by its branch (the neighbour
                 of s it hangs from) gives g = min d(u) + d(w) + 1 over the edges (u, w) of P - s joining different branches.
A sample of low-degree starts is also held equal to the DFS."""
import numpy as np
import pytest
import scipy.sparse as sp

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200 import host_mirror as hm
from fullsize_util import need, defaults
from test_zzc_var_len_trails_full_size import effective

pytestmark = pytest.mark.gpu
SCALE, EF, NSTARTS = 16, 16, 512


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def girth_through(P, u, w, s, k):
    """the levels of the BFS from s in P up to depth k (d, -1 unreached) and the shortest cycle through s that crosses branches
    (None above k), from the tree's branch labels"""
    n = P.shape[0]
    d = np.full(n, -1, np.int64)
    lab = np.full(n, -1, np.int64)
    d[s] = 0
    front = P.indices[P.indptr[s]:P.indptr[s + 1]]
    d[front] = 1
    lab[front] = front
    level = 1
    while level < k and len(front):
        sub = P[front]
        src = np.repeat(front, np.diff(sub.indptr))
        dst = sub.indices
        new = d[dst] < 0
        src, dst = src[new], dst[new]
        lab[dst] = lab[src]                                        # one parent per new vertex: a BFS tree
        front = np.unique(dst)
        d[front] = level + 1
        level += 1
    ok = (u != s) & (w != s) & (d[u] > 0) & (d[w] > 0) & (lab[u] != lab[w])
    g = (d[u][ok] + d[w][ok] + 1).min() if ok.any() else None
    return d, g


def test_reach_both_rmat_rows_and_diagonal_equal_bfs():
    need(16, 16)
    n = 1 << SCALE
    A = orc.rmat_csr(SCALE, EF, 1)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(A.p))
    cols = A.j.astype(np.uint64)
    keep = rows != cols
    rows, cols = rows[keep], cols[keep]
    rng = np.random.default_rng(23)
    extra = rng.choice(len(rows), len(rows) // 100, replace=False)
    rows, cols = np.concatenate([rows, rows[extra]]), np.concatenate([cols, cols[extra]])
    ids = np.arange(len(rows), dtype=np.uint64)
    T = hm.Tensor(n, rows, cols, ids)
    gone = rng.choice(len(rows), len(rows) // 100, replace=False)
    T.remove(ids[gone], rows[gone], cols[gone], route=hm.WRITE_DEVICE)
    ns, nd = rng.integers(0, n, 20000).astype(np.uint64), rng.integers(0, n, 20000).astype(np.uint64)
    ok = ns != nd
    old = rng.choice(len(rows), 20000)
    ns, nd = np.concatenate([ns[ok], rows[old], rows[gone[:5000]]]), np.concatenate([nd[ok], cols[old], cols[gone[:5000]]])
    T.add(ns, nd, np.arange(len(ids), len(ids) + len(ns), dtype=np.uint64), route=hm.WRITE_DEVICE)
    c = T.counts()
    assert c[0] > 0 and c[1] > 0 and c[4] > 0 and c[5] > 0, "test setup: dp, dm, me_dp and me_dm hold pending writes"
    starts = np.sort(rng.choice(n, NSTARTS, replace=False)).astype(np.uint64)
    M = effective(T, n)
    assert M.diagonal().sum() == 0
    Msum = (M + M.T).tocsr()
    P = Msum.copy()
    P.data[:] = 1
    coo = P.tocoo()
    two = np.asarray((Msum >= 2).sum(axis=1)).ravel() > 0          # two relationships to one neighbour: g = 2
    for k in (3, 4):
        R = fb.var_len_reach_both(starts, [T.layers()], 1, k)
        I, J, _ = R.extract_tuples()
        got = sp.csr_matrix((np.ones(len(I)), (I.astype(np.int64), J.astype(np.int64))), shape=(NSTARTS, n))
        closed = 0
        for i, s in enumerate(starts.astype(np.int64)):
            d, g = girth_through(P, coo.row, coo.col, s, k)
            want = set(np.flatnonzero(d > 0).tolist())
            inc = two[s] or (g is not None and g <= k)
            if inc:
                want.add(int(s))
                closed += 1
            row = set(got.indices[got.indptr[i]:got.indptr[i + 1]].tolist())
            assert row == want, (k, int(s), len(row), len(want), int(s) in row, inc)
        print(f"RMAT-{SCALE}: k = {k}: {got.nnz} (start, end) pairs, {closed} of {NSTARTS} starts on a cycle of <= {k} edges")
        assert got.nnz > 10 ** 6 and 0 < closed < NSTARTS
    # a sample of low-degree starts against the DFS: those with the fewest 3-edge walks, so that the DFS stays small
    deg = np.diff(P.indptr).astype(np.float64)
    walks3 = (P @ (P @ deg))[starts.astype(np.int64)]
    order = np.argsort(walks3)
    small = starts[order[deg[starts[order].astype(np.int64)] >= 2][:6]]
    for k in (2, 3):
        w = hm.var_len_trails([T], small, fb.DIR_BOTH, 1, k, emit_path=False, route=hm.ROUTE_BY_GET)
        row = np.repeat(np.arange(len(small)), np.diff(w["p"]).astype(np.int64))
        I, J, _ = fb.var_len_reach_both(small, [T.layers()], 1, k).extract_tuples()
        assert set(zip(I.tolist(), J.tolist())) == set(zip(row.tolist(), w["end"].tolist()))
