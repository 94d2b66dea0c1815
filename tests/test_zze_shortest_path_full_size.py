"""Full size: shortestPath over an RMAT-16 tensor built on the device with pending writes (deletes, re-adds, new pairs, new ids on
loaded pairs), 1,024 pairs, directed and undirected, max_hops 3 and unbounded, checked without the reference route.  With M the
effective multiplicity matrix (test_zzc's `effective`) and P = pattern(M), or pattern(M + M^T) when undirected: a row is Null exactly
when dist_P(src, dst) exceeds max_hops (or is infinite); otherwise its path runs from src to dst over edges of P and has
dist_P(src, dst) edges, by scipy's BFS.  A sample of low-degree pairs is held equal to the reference route."""
import numpy as np
import pytest
import scipy.sparse as sp
from scipy.sparse.csgraph import shortest_path as sp_dist

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200 import host_mirror as hm
from fullsize_util import need, defaults
from test_zzc_var_len_trails_full_size import effective

pytestmark = pytest.mark.gpu
SCALE, EF, NPAIRS = 16, 16, 1024


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def test_shortest_path_rmat_lengths_equal_bfs_distances():
    need(16, 16)
    n = 1 << SCALE
    A = orc.rmat_csr(SCALE, EF, 1)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(A.p))
    cols = A.j.astype(np.uint64)
    rng = np.random.default_rng(29)
    extra = rng.choice(len(rows), len(rows) // 100, replace=False)
    rows, cols = np.concatenate([rows, rows[extra]]), np.concatenate([cols, cols[extra]])
    ids = np.arange(len(rows), dtype=np.uint64)
    T = hm.Tensor(n, rows, cols, ids)
    gone = rng.choice(len(rows), len(rows) // 50, replace=False)
    T.remove(ids[gone], rows[gone], cols[gone], route=hm.WRITE_DEVICE)
    ns, nd = rng.integers(0, n, 20000).astype(np.uint64), rng.integers(0, n, 20000).astype(np.uint64)
    old = rng.choice(len(rows), 20000)
    ns, nd = np.concatenate([ns, rows[old], rows[gone[:5000]]]), np.concatenate([nd, cols[old], cols[gone[:5000]]])
    T.add(ns, nd, np.arange(len(ids), len(ids) + len(ns), dtype=np.uint64), route=hm.WRITE_DEVICE)
    c = T.counts()
    assert c[0] > 0 and c[1] > 0, "test setup: dp and dm hold pending writes"
    M = effective(T, n)
    live = np.flatnonzero(np.asarray((M + M.T).sum(axis=1)).ravel() > 0)
    srcs = rng.choice(live, NPAIRS).astype(np.uint64)
    dsts = rng.choice(live, NPAIRS).astype(np.uint64)
    srcs[:8] = dsts[:8]                                            # src == dst rows
    for directed in (True, False):
        P = M.copy() if directed else (M + M.T).tocsr()
        P.data[:] = 1
        P = P.tocsr()
        D = sp_dist(P, method="D", unweighted=True, indices=np.unique(srcs).astype(np.int64))
        row_of = {int(s): k for k, s in enumerate(np.unique(srcs))}
        for hi in (3, None):
            for lo in (0, 1):
                got = hm.shortest_path(None, [T], [T], srcs, dsts, directed, lo, hi, route=hm.SP_DEVICE)
                found = 0
                for s, d, x in zip(srcs.tolist(), dsts.tolist(), got):
                    dist = D[row_of[s], d]
                    if s == d:
                        assert (x is not None) == (lo == 0) and (x is None or x[0] == [s])
                        continue
                    if not np.isfinite(dist) or (hi is not None and dist > hi):
                        assert x is None, (s, d, dist)
                        continue
                    nodes, rel = x
                    assert nodes[0] == s and nodes[-1] == d and len(nodes) - 1 == dist, (s, d, dist, nodes)
                    assert all(P[a, b] for a, b in zip(nodes, nodes[1:]))
                    assert len(rel) == len(nodes) - 1
                    found += 1
                print(f"RMAT-{SCALE}: directed={directed} min={lo} max={hi}: {found} of {NPAIRS} paths")
                assert found > NPAIRS // 10
    # low-degree pairs against the reference route
    Psym = (M + M.T).tocsr()
    deg = np.diff(Psym.indptr)
    small = np.flatnonzero((deg >= 1) & (deg <= 3))[:64].astype(np.uint64)
    pairs_s, pairs_d = small[:32], small[32:64]
    for directed in (True, False):
        for hi in (4, None):
            dev = hm.shortest_path(None, [T], [T], pairs_s, pairs_d, directed, 1, hi, route=hm.SP_DEVICE)
            ref = hm.shortest_path(None, [T], [T], pairs_s, pairs_d, directed, 1, hi, route=hm.SP_BY_ITER)
            assert dev == ref
