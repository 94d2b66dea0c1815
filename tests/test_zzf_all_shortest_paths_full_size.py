"""Full size: allShortestPaths over two RMAT-16 relationship types built on the device with pending writes (deletes, re-adds, new
pairs, new ids on loaded pairs), 1,024 random pairs, Out and Both, checked without the reference route.  With W the sum of the two
types' effective multiplicity matrices (test_zzc's `effective`; Both: W + W^T with a self-loop once): each pair's path length is
its BFS distance in pattern(W) (for src == dst, the shortest cycle through it), and its count is an independent count of the
shortest walks, the level DP over W restricted to the nodes on a shortest path, in exact Python integers (saturated at
2^64 - 1).  For pairs with at most 10^4 paths, the listed paths are valid, distinct and of that length."""
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
SAT = (1 << 64) - 1


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def rmat_tensor(n, seed, id0):
    A = orc.rmat_csr(SCALE, EF, seed)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(A.p))
    cols = A.j.astype(np.uint64)
    rng = np.random.default_rng(seed)
    extra = rng.choice(len(rows), len(rows) // 100, replace=False)
    rows, cols = np.concatenate([rows, rows[extra]]), np.concatenate([cols, cols[extra]])
    ids = np.arange(id0, id0 + len(rows), dtype=np.uint64)
    T = hm.Tensor(n, rows, cols, ids)
    gone = rng.choice(len(rows), len(rows) // 50, replace=False)
    T.remove(ids[gone], rows[gone], cols[gone], route=hm.WRITE_DEVICE)
    ns, nd = rng.integers(0, n, 20000).astype(np.uint64), rng.integers(0, n, 20000).astype(np.uint64)
    old = rng.choice(len(rows), 20000)
    ns, nd = np.concatenate([ns, rows[old], rows[gone[:5000]]]), np.concatenate([nd, cols[old], cols[gone[:5000]]])
    T.add(ns, nd, np.arange(id0 + len(ids), id0 + len(ids) + len(ns), dtype=np.uint64), route=hm.WRITE_DEVICE)
    c = T.counts()
    assert c[0] > 0 and c[1] > 0, "test setup: dp and dm hold pending writes"
    return T


def dag_count(W, WT, df, db, s, d):
    """shortest s -> d walks in the multigraph W (d == s: shortest closed walks), exact: the level DP over the nodes with
    df + db == the distance, counts summed over W's entries (multiplicities)"""
    if s == d:
        ins = WT.indices[WT.indptr[s]:WT.indptr[s + 1]]
        ok = [u for u in ins if np.isfinite(df[u])]
        if not ok:
            return 0, 0
        L = int(min(df[u] for u in ok)) + 1
        ends = {u: int(WT[s, u]) for u in ok if df[u] == L - 1}
    else:
        if not np.isfinite(df[d]):
            return 0, 0
        L = int(df[d])
        ends = None
    ondag = np.isfinite(df) & np.isfinite(db) & (df + db == L)
    ondag[s] = True
    on = [[] for _ in range(L + 1)]
    for v in np.flatnonzero(ondag):
        on[int(df[v])].append(int(v))
    cnt = {s: 1}
    for l in range(1, (L - 1 if s == d else L) + 1):
        for v in on[l]:
            us, ws = WT.indices[WT.indptr[v]:WT.indptr[v + 1]], WT.data[WT.indptr[v]:WT.indptr[v + 1]]
            keep = (df[us] == l - 1) & ondag[us]
            cnt[v] = sum(cnt[int(u)] * int(w) for u, w in zip(us[keep], ws[keep]))
    if s == d:
        total = sum(cnt.get(u, 0) * w for u, w in ends.items())
    else:
        total = cnt.get(d, 0)
    return min(total, SAT), L


def test_all_shortest_paths_rmat_counts_and_lengths():
    need(16, 16)
    n = 1 << SCALE
    types = [rmat_tensor(n, 1, 0), rmat_tensor(n, 2, 1 << 40)]
    W = (effective(types[0], n) + effective(types[1], n)).tocsr().astype(np.int64)
    rng = np.random.default_rng(31)
    live = np.flatnonzero(np.asarray((W + W.T).sum(axis=1)).ravel() > 0)
    srcs = rng.choice(live, NPAIRS).astype(np.uint64)
    dsts = rng.choice(live, NPAIRS).astype(np.uint64)
    srcs[:8] = dsts[:8]                                            # shortest cycles
    for directed in (True, False):
        G = W if directed else (W + W.T - sp.diags(W.diagonal(), dtype=np.int64)).tocsr()
        G.eliminate_zeros()
        GT = G.T.tocsr()
        P = G.copy()
        P.data[:] = 1
        us, ud = np.unique(srcs), np.unique(dsts)
        DF = sp_dist(P, method="D", unweighted=True, indices=us.astype(np.int64))
        DB = sp_dist(P.T.tocsr(), method="D", unweighted=True, indices=ud.astype(np.int64))
        rf, rb = {int(s): k for k, s in enumerate(us)}, {int(d): k for k, d in enumerate(ud)}
        got = fb.all_shortest_paths(srcs, dsts, [t.layers() for t in types], fb.DIR_OUT if directed else fb.DIR_BOTH, edge_capacity=0)
        found = listed = 0
        small = []
        for i, (s, d) in enumerate(zip(srcs.tolist(), dsts.tolist())):
            c, L = dag_count(G, GT, DF[rf[s]], DB[rb[d]], s, d)
            assert int(got["count"][i]) == c and int(got["len"][i]) == (L if c else 0), (i, s, d, c, L, got["count"][i], got["len"][i])
            found += c > 0
            if 0 < c <= 10 ** 4:
                small.append(i)
        assert found > NPAIRS // 2
        sel = small[:256]
        out = fb.all_shortest_paths(srcs[sel], dsts[sel], [t.layers() for t in types], fb.DIR_OUT if directed else fb.DIR_BOTH)
        e = k = 0
        for j, i in enumerate(sel):
            c, L = int(out["count"][j]), int(out["len"][j])
            seen = set()
            for _ in range(c):
                edges = tuple(out["edges"][e:e + L].tolist())
                nodes = out["nodes"][e + k:e + k + L + 1].tolist()
                assert nodes[0] == srcs[i] and nodes[-1] == dsts[i] and len(edges) == L
                walk = nodes[::-1] if srcs[i] == dsts[i] else nodes          # a cycle's list starts with its closing edge
                assert all(G[a, b] > 0 for a, b in zip(walk, walk[1:])), (i, nodes)
                seen.add((edges, tuple(nodes)))
                e += L
                k += 1
            assert len(seen) == c
            listed += c
        print(f"RMAT-{SCALE} x 2 types: directed={directed}: {found} of {NPAIRS} pairs connected, {listed} paths listed and checked")
