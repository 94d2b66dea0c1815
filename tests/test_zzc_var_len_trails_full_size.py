"""Full size: B200_var_len_trails on a self-loop-free RMAT tensor built on the device (Tensor::bulk_load, 1 % of pairs with a second
edge) with pending writes (deletes, re-adds, new pairs, new ids on loaded pairs), checked against linear algebra rather than the
DFS.  With M the effective multiplicity matrix (ids per pair over (m \\ dm) u dp and (me \\ me_dm) u me_dp), built by scipy from the
layers, and no self-loops, a trail of 2 edges is any 2-walk and a 3-walk repeats an edge only as s -> u -> s -> u (edge 1 = edge 3):
  count mode     trails_2 = M^2 1,  trails_3 = M^3 1 - (M o M^T) 1   per start;
  endpoints mode per (start s, end t) at hop 3: M^3[s, t] - M[s, t] M[t, s].
A sample of starts is also held equal to the DFS list for list."""
import numpy as np
import pytest
import scipy.sparse as sp

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200 import host_mirror as hm
from fullsize_util import need, defaults

pytestmark = pytest.mark.gpu
# RMAT-16, edge factor 16: 512 random starts have about 1.1e9 trails of 3 edges.  The stored tree (the trails of 1 and 2 edges)
# holds about 4e6 entries (0.1 GB); the last level's candidate flags and positions (12 bytes each) take about 13 GB.
SCALE, EF, NSTARTS, NENDS = 16, 16, 512, 96
MULTI = (1 << 64) - 1


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def effective(t, n):
    """M from the nine layers: the pair's value by Tensor::eff_get, a MULTI_EDGE value counting its merged id list"""
    L = t.tuples()
    key = lambda r, c: (r.astype(np.uint64) << np.uint64(32)) | c.astype(np.uint64)
    km, kdp, kdm = key(*L[0][:2]), key(*L[1][:2]), key(*L[2][:2])
    keep = ~np.isin(km, kdm) & ~np.isin(km, kdp)
    k = np.concatenate([km[keep], kdp])
    v = np.concatenate([L[0][2][keep], L[1][2]])
    pair = lambda x: np.stack([x[0], x[1]], 1)
    me, medp, medm = pair(L[6]), pair(L[7]), pair(L[8])
    gone = set(map(tuple, medm.tolist()))                            # (me \ me_dm) u me_dp on (key, id)
    live = np.array([r for r in me.tolist() if tuple(r) not in gone], np.uint64).reshape(-1, 2)
    ids = np.unique(np.concatenate([live, medp]), axis=0)
    uk, cnt = np.unique(ids[:, 0], return_counts=True)
    mult = np.ones(len(k))
    multi = v == np.uint64(MULTI)
    pos = np.searchsorted(uk, k[multi])
    assert (uk[pos] == k[multi]).all(), "a MULTI_EDGE pair without ids"
    mult[multi] = cnt[pos]
    r, c = (k >> np.uint64(32)).astype(np.int64), (k & np.uint64(0xFFFFFFFF)).astype(np.int64)
    return sp.csr_matrix((mult, (r, c)), shape=(n, n))


def test_trails_rmat_counts_and_endpoints_equal_linear_algebra():
    need(24, 24)
    n = 1 << SCALE
    A = orc.rmat_csr(SCALE, EF, 1)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(A.p))
    cols = A.j.astype(np.uint64)
    keep = rows != cols
    rows, cols = rows[keep], cols[keep]
    rng = np.random.default_rng(21)
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
    L = [T.layers()]
    r2 = fb.var_len_trails(starts, L, fb.DIR_OUT, 2, 2, mode="count")
    r3 = fb.var_len_trails(starts, L, fb.DIR_OUT, 3, 3, mode="count")
    e3 = fb.var_len_trails(starts[:NENDS], L, fb.DIR_OUT, 3, 3, mode="ends")
    M = effective(T, n)
    assert M.diagonal().sum() == 0
    one = np.ones(n)
    d1 = M @ one
    d2 = M @ d1
    d3 = M @ d2
    back = np.asarray(M.multiply(M.T).sum(axis=1)).ravel()
    print(f"RMAT-{SCALE} ef {EF}: {M.nnz} pairs, {NSTARTS} starts: {int(d1[starts].sum())} trails of 1 edge (stored), "
          f"{r2['nout']} of 2 (stored), {r3['nout']} of 3")
    assert np.array_equal(np.diff(r2["p"]).astype(np.float64), d2[starts])
    assert np.array_equal(np.diff(r3["p"]).astype(np.float64), d3[starts] - back[starts])
    assert r3["npath"] == 3 * r3["nout"] and r3["nout"] > 10 ** 8
    # endpoints: per (start, end) pair
    S = sp.csr_matrix((np.ones(NENDS), (np.arange(NENDS), starts[:NENDS].astype(np.int64))), shape=(NENDS, n))
    W = ((S @ M) @ M) @ M - S @ M.multiply(M.T)
    W.eliminate_zeros()
    row = np.repeat(np.arange(NENDS), np.diff(e3["p"]).astype(np.int64))
    got = sp.csr_matrix((np.ones(len(row)), (row, e3["end"].astype(np.int64))), shape=(NENDS, n))
    got.sum_duplicates()
    assert (abs(got - W)).sum() == 0
    assert (e3["hops"] == 3).all()
    # a sample of starts, list for list against the DFS
    small = starts[np.argsort(d3[starts])[:6]]
    for lo, hi in ((1, 3), (3, 3)):
        want = hm.var_len_trails([T], small, fb.DIR_OUT, lo, hi, route=hm.ROUTE_BY_GET)
        have = hm.var_len_trails([T], small, fb.DIR_OUT, lo, hi, route=hm.ROUTE_DEVICE)
        for k in ("p", "end", "hops", "edges", "nodes"):
            assert np.array_equal(want[k], have[k]), k
