"""CPU-side checks of B200_var_len_reach_both.  First the algorithm itself, restated in Python (the reach over A u A' for v != s;
for the start, the run test on its sorted adjacency and the bit-split BFS in G' - s), against brute-force enumeration of
bidirectional trails over relationship ids on random multigraphs with self-loops, reciprocal pairs and multi-edges; the plain walk
reach over A u A' is shown to be wrong for the start.  Then the argument, domain, dimension and index errors, empty batches and
windows with no device work, and without a GPU a loud failure before any host work.  No kernel is launched here."""
import ctypes as C
from collections import deque

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, P
from falkordb_b200.grb import Matrix, TensorLayers, TENSOR_LAYERS

INF = None
WINDOWS = [(lo, hi) for lo in (0, 1) for hi in list(range(7)) + [INF]]


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def trail_ends(n, edges, s):
    """brute force: {(end, hops)} over every relationship-unique walk from s, edges (u, v, id) read both ways, a self-loop once"""
    inc = [[] for _ in range(n)]
    for u, v, i in edges:
        inc[u].append((v, i))
        if v != u:
            inc[v].append((u, i))
    out = {(s, 0)}
    stack, seen = [(s, frozenset())], set()                         # a (node, used ids) state continues the same way every time
    while stack:
        x, used = stack.pop()
        for y, i in inc[x]:
            if i in used:
                continue
            u2 = used | {i}
            out.add((y, len(u2)))
            if (y, u2) not in seen:
                seen.add((y, u2))
                stack.append((y, u2))
    return out


def brute(n, edges, s, lo, hi):
    return {v for v, h in trail_ends(n, edges, s) if h >= lo and (hi is INF or h <= hi)}


def sym_adj(n, edges):
    adj = [set() for _ in range(n)]
    for u, v, _ in edges:
        adj[u].add(v)
        adj[v].add(u)
    return adj


def bfs_levels(adj, seeds, reached, limit, stop=lambda f: False):
    """masked levels F<!R> = F.S, R |= F from `seeds` with R = `reached`; returns True as soon as stop(F) holds"""
    F, R, level = set(seeds), set(reached), 0
    while F and (limit is INF or level < limit):
        F = {y for x in F for y in adj[x]} - R
        if stop(F):
            return True
        R |= F
        level += 1
    return False


def restated(n, edges, s, lo, hi):
    """steps 1-4 of B200_var_len_reach_both"""
    adj = sym_adj(n, edges)
    # 1. the reach over A u A' with the start included and never re-expanded: exact for v != s
    dist = {s: 0}
    q = deque([s])
    while q:
        x = q.popleft()
        for y in adj[x]:
            if y not in dist:
                dist[y] = dist[x] + 1
                q.append(y)
    got = {v for v, d in dist.items() if v != s and (hi is INF or d <= hi)}
    if lo == 0:
        return got | {s}
    if hi == 0:
        return got
    # 2. the start's adjacency under Both, one entry per relationship, a self-loop once: sorted neighbours and their runs
    nb = sorted([v for u, v, _ in edges if u == s] + [u for u, v, _ in edges if v == s and u != s])
    runs = {}
    for c in nb:
        runs[c] = runs.get(c, 0) + 1
    g1 = s in runs
    g2 = any(c != s and k >= 2 for c, k in runs.items())
    inc = g1 or (g2 and (hi is INF or hi >= 2))
    # 3. longer cycles: one row per bit of the ranks of the distinct neighbours c != s, k - 2 masked levels in G' - s
    cs = [c for c in sorted(runs) if c != s]
    if not inc and (hi is INF or hi >= 3) and len(cs) >= 2:
        for b in range(int(len(cs) - 1).bit_length()):
            X0 = {c for r, c in enumerate(cs) if not (r >> b) & 1}
            T = {c for r, c in enumerate(cs) if (r >> b) & 1}
            if bfs_levels(adj, X0, X0 | {s}, INF if hi is INF else hi - 2, lambda F: bool(F & T)):
                inc = True
                break
    # 4. the fix-up of the start's own entry
    return got | {s} if inc else got


def walk_reach(n, edges, s, lo, hi):
    """the plain reach over A u A': every vertex at the end of a walk of lo..hi edges (the negative control)"""
    adj = sym_adj(n, edges)
    out = {s} if lo == 0 else set()
    F, level = {s}, 0
    seen = set()
    while F and (hi is INF or level < hi):
        F = {y for x in F for y in adj[x]}
        key = frozenset(F)
        if key in seen:
            break
        seen.add(key)
        out |= F
        level += 1
    return out


def random_multigraph(rng):
    n = int(rng.integers(1, 10))
    m = int(rng.integers(0, 12))
    edges = []
    for i in range(m):
        kind = rng.random()
        if kind < 0.12:
            v = int(rng.integers(0, n))
            edges.append((v, v, i))                                  # a self-loop
        elif kind < 0.25 and edges:
            u, v, _ = edges[int(rng.integers(0, len(edges)))]
            edges.append((v, u, i) if rng.random() < 0.5 else (u, v, i))   # a reciprocal pair or a multi-edge pair
        else:
            edges.append((int(rng.integers(0, n)), int(rng.integers(0, n)), i))
    return n, edges


def test_restated_algorithm_equals_brute_force_trails():
    rng = np.random.default_rng(2026)
    graphs = cases = closed = 0
    control_differs = False
    while graphs < 2400:
        n, edges = random_multigraph(rng)
        graphs += 1
        for s in range(n):
            ends = trail_ends(n, edges, s)
            for lo, hi in WINDOWS:
                want = {v for v, h in ends if h >= lo and (hi is INF or h <= hi)}
                assert restated(n, edges, s, lo, hi) == want, (n, edges, s, lo, hi)
                control_differs |= walk_reach(n, edges, s, lo, hi) != want
                cases += 1
                closed += lo == 1 and s in want
    assert graphs >= 2000 and cases > 100000 and closed > 1000
    assert control_differs, "the walk reach over A u A' should be wrong for some start"


def test_the_walk_reach_is_wrong_for_the_start():
    edges = [(0, 1, 0), (1, 2, 1)]                                   # a path: no cycle, but s - 1 - s is a walk
    assert 0 in walk_reach(3, edges, 0, 1, 2)
    assert brute(3, edges, 0, 1, 2) == restated(3, edges, 0, 1, 2) == {1, 2}
    tri = [(0, 1, 0), (1, 2, 1), (2, 0, 2)]                          # a triangle closes at 3 hops, not 2
    assert restated(3, tri, 0, 1, 2) == brute(3, tri, 0, 1, 2) == {1, 2}
    assert restated(3, tri, 0, 1, 3) == brute(3, tri, 0, 1, 3) == {0, 1, 2}


def call(starts, types, ntypes=None, lo=1, hi=3, out=True):
    starts = np.ascontiguousarray(starts, dtype=np.uint64)
    ls = (TensorLayers * max(1, len(types or ())))()
    for k, t in enumerate(types or ()):
        for name in TENSOR_LAYERS:
            x = t.get(name)
            setattr(ls[k], name, None if x is None else x.h)
    h = P()
    info = lib().B200_var_len_reach_both(C.byref(h) if out else None, starts.ctypes.data if len(starts) else None, len(starts),
                                         None if types is None else ls, len(types or ()) if ntypes is None else ntypes, lo, hi)
    R = Matrix(0, 0, bool, _handle=h) if h.value else None
    return info, R


def tensor(n=16, huge=False):
    nn = 1 << 60 if huge else n
    return {"m": Matrix(nn, nn, "u64"), "dp": Matrix(nn, nn, "u64"), "dm": Matrix(nn, nn), "mt": Matrix(nn, nn),
            "mt_dp": Matrix(nn, nn), "mt_dm": Matrix(nn, nn), "me": Matrix(1 << 60, 1 << 60), "me_dp": Matrix(1 << 60, 1 << 60),
            "me_dm": Matrix(1 << 60, 1 << 60)}


def test_null_pointers():
    fb.init()
    t = tensor()
    assert call([0], [t], out=False)[0] == -2                               # GrB_NULL_POINTER: reached
    assert call([0], None, ntypes=1)[0] == -2                               # types
    assert call([0], [dict(t, m=None)])[0] == -2                            # m
    assert call([0], [dict(t, mt=None)])[0] == -2                           # mt
    ls = (TensorLayers * 1)()
    ls[0].m, ls[0].mt = t["m"].h, t["mt"].h
    h = P()
    assert lib().B200_var_len_reach_both(C.byref(h), None, 2, ls, 1, 1, 2) == -2     # starts


def test_values_domains_dimensions_indices_and_windows():
    fb.init()
    t, small = tensor(), tensor(8)
    assert call([0], [t], ntypes=0)[0] == -3                                # GrB_INVALID_VALUE: ntypes < 1
    assert call([0], [t], ntypes=65537)[0] == -3
    assert call([0], [dict(t, m=Matrix(16, 16))])[0] == -5                  # GrB_DOMAIN_MISMATCH: m not UINT64
    assert call([0], [dict(t, dp=Matrix(16, 16))])[0] == -5                 # dp not UINT64
    assert call([0], [dict(t, m=Matrix(16, 8, "u64"))])[0] == -6            # GrB_DIMENSION_MISMATCH
    assert call([0], [t, small])[0] == -6
    for k in ("dp", "dm", "mt", "mt_dp", "mt_dm"):
        assert call([0], [dict(t, **{k: small[k]})])[0] == -6, k
    assert call([16], [t])[0] == -4                                         # GrB_INVALID_INDEX: a start >= n
    assert call([0], [tensor(huge=True)])[0] == -8                          # GrB_NOT_IMPLEMENTED: host-resident layers
    for lo in (2, 3):
        assert call([0], [t], lo=lo, hi=5)[0] == -8                         # min_hops > 1 keeps the trail enumerator


def test_empty_batches_and_windows_do_no_device_work():
    fb.init()
    t = tensor()
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    info, R = call([], [t])
    assert info == 0 and (R.nrows(), R.ncols(), R.nvals()) == (0, 16, 0)
    info, R = call([0, 5, 5], [t], lo=1, hi=0)                              # min_hops > max_hops
    assert info == 0 and (R.nrows(), R.ncols(), R.nvals()) == (3, 16, 0)
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_var_len_reach_both_fails_loudly_without_gpu():
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    for lo, hi in ((0, 0), (1, 1), (1, 3), (0, (1 << 64) - 1)):
        assert call([0, 1], [t, t], lo=lo, hi=hi)[0] == -7002               # GxB_GPU_ERROR
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before
    assert t["m"].pending()                                                 # the queued write was not finished by the call
    with pytest.raises(fb.GrbError) as e:
        fb.var_len_reach_both([0], [t])
    assert e.value.info == -7002
