"""CPU-side checks of shortestPath.  The reference's bidirectional BFS (bfs_shortest_path, eval.rs:1386-1513) is transcribed in
Python and held to the flow test's 5-node graph and expectations (tests/golden/shortest_path_flow_cases.json).  The
level-synchronous statement B200_shortest_path implements (parent = lowest-ranked front neighbour, next front by (parent rank, v),
meet = least (od, parent rank, v)), with fronts cut into rank-ordered pieces of any size, is held equal to the transcription path for
path on random multigraphs with self-loops, reciprocal pairs and multi-edges, typed and untyped, directed and undirected, and every
found path is checked for validity and BFS length.  The host mirror's reference route (shortest_path_by_iter) runs here over the
adjacency VersionedMatrix with pending writes, which needs no device, and is held to the transcription.  Then the argument errors,
npairs == 0 with no device work, and without a GPU a loud failure before any host work."""
import ctypes as C
import json
import os
from collections import deque

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Matrix

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "shortest_path_flow_cases.json")
INF = None


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def sides(n, types, named, directed, adj=None):
    """each side's sorted neighbour lists (NeighborIter::new / new_reversed).  types: {name: [(u, v, id)]} effective
    relationships; named: the pattern's type names (missing ones dropped), [] for untyped; adj: the adjacency pairs (untyped)"""
    present = [types[t] for t in named if t in types] if named else list(types.values())
    out_, in_ = [set() for _ in range(n)], [set() for _ in range(n)]
    for rels in present:
        for u, v, _ in rels:
            out_[u].add(v)
            in_[v].add(u)
    if not named:
        out_ = [set() for _ in range(n)]
        for u, v in (adj if adj is not None else {(u, v) for rels in types.values() for u, v, _ in rels}):
            out_[u].add(v)
    if directed:
        return [sorted(x) for x in out_], [sorted(x) for x in in_]
    both = [sorted(out_[u] | in_[u]) for u in range(n)]
    return both, both


def bfs_shortest_path(fwd, bwd, src, dst, max_level, min_hops):
    """eval_shortest_path + bfs_shortest_path, statement for statement; max_level None: unbounded"""
    if min_hops == 0 and src == dst:
        return [src]
    if src == dst:
        return None
    max_level = float("inf") if max_level is None else max_level
    f_map, b_map = {src: (src, 0)}, {dst: (dst, 0)}
    f_front, b_front = [src], [dst]
    df = db = 0
    meet = None
    while meet is None:
        if not f_front or not b_front or df + db >= max_level:
            return None
        expand_fwd = len(f_front) <= len(b_front)
        front, own, other, nbrs = (f_front, f_map, b_map, fwd) if expand_fwd else (b_front, b_map, f_map, bwd)
        depth = (df if expand_fwd else db) + 1
        nxt = []
        for cur in front:
            for nb in nbrs[cur]:
                if nb not in own:
                    own[nb] = (cur, depth)
                    if nb in other:
                        od = other[nb][1]
                        if meet is None or od < meet[0]:
                            meet = (od, nb)
                    else:
                        nxt.append(nb)
        if expand_fwd:
            f_front, df = nxt, depth
        else:
            b_front, db = nxt, depth
    return reconstruct(f_map, b_map, meet[1], src, dst, min_hops)


def reconstruct(f_map, b_map, m, src, dst, min_hops):
    path, cur = [m], m
    while cur != src:
        cur = f_map[cur][0]
        path.append(cur)
    path.reverse()
    cur = m
    while cur != dst:
        cur = b_map[cur][0]
        path.append(cur)
    return None if len(path) - 1 < min_hops else path


def level_sync(fwd, bwd, src, dst, max_level, min_hops, budget=None):
    """what shortest_path.cu computes: per round, each piece of the front (rank-ordered, at most `budget` neighbour entries unless
    one node has more) emits (v, r) for unseen v, keeps the least r per v, marks them seen; the meet is the least (od, r, v), replaced
    by a later piece only with a strictly smaller od; the next front is the survivors by (r, v)"""
    if min_hops == 0 and src == dst:
        return [src]
    if src == dst:
        return None
    max_level = float("inf") if max_level is None else max_level
    maps, fronts, dep = [{src: (src, 0)}, {dst: (dst, 0)}], [[src], [dst]], [0, 0]
    while True:
        if not fronts[0] or not fronts[1] or dep[0] + dep[1] >= max_level:
            return None
        sd = 0 if len(fronts[0]) <= len(fronts[1]) else 1
        nbrs, own, other, front = (fwd, bwd)[sd], maps[sd], maps[1 - sd], fronts[sd]
        best, nxt, i0 = None, [], 0
        while i0 < len(front):
            i1, tot = i0, 0
            while i1 < len(front) and (i1 == i0 or budget is None or tot + len(nbrs[front[i1]]) <= budget):
                tot += len(nbrs[front[i1]])
                i1 += 1
            first = {}
            for r in range(i0, i1):
                for v in nbrs[front[r]]:
                    if v not in own and v not in first:
                        first[v] = r
            cands, surv = [], []
            for v, r in first.items():
                own[v] = (front[r], dep[sd] + 1)
                (cands.append((other[v][1], r, v)) if v in other else surv.append((r, v)))
            if cands and (best is None or min(cands)[0] < best[0]):
                best = min(cands)
            nxt += [v for _, v in sorted(surv)]
            i0 = i1
        fronts[sd] = nxt
        dep[sd] += 1
        if best is not None:
            return reconstruct(maps[0], maps[1], best[2], src, dst, min_hops)


def bfs_dist(fwd, src):
    dist = {src: 0}
    q = deque([src])
    while q:
        u = q.popleft()
        for v in fwd[u]:
            if v not in dist:
                dist[v] = dist[u] + 1
                q.append(v)
    return dist


def random_graph(rng, n, ntypes):
    types, nid = {}, 0
    for t in range(ntypes):
        m = int(rng.integers(0, 3 * n))
        rels = []
        for _ in range(m):
            u, v = int(rng.integers(0, n)), int(rng.integers(0, n))
            k = 1 + int(rng.random() < 0.2)                        # multi-edges
            for _ in range(k):
                rels.append((u, v, nid))
                nid += 1
            if rng.random() < 0.15:
                rels.append((v, u, nid))                           # reciprocal pairs
                nid += 1
        if rng.random() < 0.5 and n:
            x = int(rng.integers(0, n))
            rels.append((x, x, nid))                               # self-loops
            nid += 1
        types[f"T{t}"] = rels
    return types


def check_path(path, fwd, src, dst, min_hops, max_hops):
    dist = bfs_dist(fwd, src)
    reach = dst in dist and (src != dst or min_hops == 0)
    d = 0 if src == dst else dist.get(dst)
    if not reach or (max_hops is not None and d > max_hops):
        assert path is None, (src, dst, path)
        return
    assert path is not None and path[0] == src and path[-1] == dst and len(path) - 1 == d, (src, dst, path, d)
    for a, b in zip(path, path[1:]):
        assert b in fwd[a]


def test_transcription_against_the_flow_goldens():
    g = json.load(open(GOLDEN))
    types = {k: [tuple(r) for r in v] for k, v in g["types"].items()}
    for c in g["cases"]:
        fwd, bwd = sides(g["n"], types, c["named"], c["directed"])
        got = [bfs_shortest_path(fwd, bwd, s, d, c["max_hops"], c["min_hops"]) for s, d in zip(c["src"], c["dst"])]
        assert got == c["nodes"], c["name"]
        got = [level_sync(fwd, bwd, s, d, c["max_hops"], c["min_hops"], 1) for s, d in zip(c["src"], c["dst"])]
        assert got == c["nodes"], c["name"]


def test_level_synchronous_pieces_equal_the_sequential_loop():
    rng = np.random.default_rng(7)
    graphs = 0
    for it in range(1200):
        n = int(rng.integers(1, 24))
        types = random_graph(rng, n, int(rng.integers(1, 4)))
        named = [] if it % 3 == 0 else [t for t in list(types) + ["MISSING"] if rng.random() < 0.7]
        for directed in (True, False):
            fwd, bwd = sides(n, types, named, directed)
            sym = sides(n, types, named, False)[0]
            pairs = [(int(rng.integers(0, n)), int(rng.integers(0, n))) for _ in range(6)] + [(0, 0)]
            for s, d in pairs:
                for lo, hi in ((1, INF), (0, INF), (1, 1), (1, 2), (0, 3), (1, 0)):
                    want = bfs_shortest_path(fwd, bwd, s, d, hi, lo)
                    for budget in (None, 1, 2, 5):
                        assert level_sync(fwd, bwd, s, d, hi, lo, budget) == want, (it, directed, s, d, lo, hi, budget)
                    check_path(want, fwd if directed else sym, s, d, lo, hi)
        graphs += 1
    assert graphs >= 1000


def test_ties_meet_on_od_then_encounter_order():
    # layered complete bipartite: every path has the same length, the meet and parents follow (od, rank, v)
    n, layers = 12, [[0], [1, 2, 3], [4, 5, 6], [7, 8], [9]]
    types = {"E": [(u, v, 100 * u + v) for a, b in zip(layers, layers[1:]) for u in a for v in b]}
    for directed in (True, False):
        fwd, bwd = sides(n, types, ["E"], directed)
        for budget in (None, 1, 3):
            assert level_sync(fwd, bwd, 0, 9, None, 1, budget) == bfs_shortest_path(fwd, bwd, 0, 9, None, 1) == [0, 1, 4, 7, 9]


def test_reference_route_over_the_adjacency_equals_the_transcription():
    """shortest_path_by_iter walks only the adjacency VersionedMatrix when no type is named and the graph has no Tensor: no device"""
    rng = np.random.default_rng(3)
    for it in range(60):
        n = int(rng.integers(2, 20))
        adj = hm.VersionedMatrix(n)
        pairs = {(int(rng.integers(0, n)), int(rng.integers(0, n))) for _ in range(int(rng.integers(0, 3 * n)))}
        if pairs:
            r, c = zip(*sorted(pairs))
            adj.set_all(r, c)
        eff = set(pairs)
        for u, v in list(pairs)[: len(pairs) // 3]:                  # pending deletes
            adj.remove(u, v)
            eff.discard((u, v))
        for _ in range(3):                                              # pending inserts
            u, v = int(rng.integers(0, n)), int(rng.integers(0, n))
            adj.set(u, v)
            eff.add((u, v))
        srcs = [int(x) for x in rng.integers(0, n, 8)] + [1]
        dsts = [int(x) for x in rng.integers(0, n, 8)] + [1]
        for directed in (True, False):
            for lo, hi in ((1, INF), (0, 2), (1, 1)):
                got = hm.shortest_path(adj, [], [], srcs, dsts, directed, lo, hi, route=hm.SP_BY_ITER)
                fwd_out = [sorted({v for u, v in eff if u == x}) for x in range(n)]
                # no relationship type, so no matrix_t: a directed pattern's backward side is empty, an undirected one walks the
                # adjacency's out-rows on both sides
                fwd, bwd = (fwd_out, [[] for _ in range(n)] if directed else fwd_out)
                want = [bfs_shortest_path(fwd, bwd, s, d, hi, lo) for s, d in zip(srcs, dsts)]
                assert [None if x is None else x[0] for x in got] == want, (it, directed, lo, hi)
                assert all(x is None or x[1] == [] for x in got)


def test_missing_types_only_zero_hop_rows():
    got = hm.shortest_path(None, [], [None], [0, 2, 3], [0, 2, 4], True, 0, None, route=hm.SP_BY_ITER)
    assert got == [([0], []), ([2], []), None]
    got = hm.shortest_path(None, [], [None, None], [0, 3], [0, 4], False, 1, None, route=hm.SP_DEVICE)
    assert got == [None, None]


def call(src, dst, fwd, bwd, lo=1, hi=(1 << 64) - 1, cap=64, nf=None, nb=None, out=True):
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    s, d = np.asarray(src, np.uint64), np.asarray(dst, np.uint64)
    p = np.zeros(len(s) + 1, np.uint64)
    nodes = np.zeros(max(cap, 1), np.uint32)
    nn = U64(0)
    f = [x[0] for x in fwd], [x[1] for x in fwd], [x[2] for x in fwd]
    b = [x[0] for x in bwd], [x[1] for x in bwd], [x[2] for x in bwd]
    info = lib().B200_shortest_path(s.ctypes.data if len(s) else None, d.ctypes.data if len(d) else None, len(s),
                                    arr(f[0]), arr(f[1]), arr(f[2]), len(fwd) if nf is None else nf,
                                    arr(b[0]), arr(b[1]), arr(b[2]), len(bwd) if nb is None else nb, lo, hi,
                                    p.ctypes.data if out else None, nodes.ctypes.data, cap, C.byref(nn))
    return info, p, nodes[: nn.value], nn.value


def op(n=16, huge=False):
    nn = 1 << 60 if huge else n
    return (Matrix(nn, nn, "u64"), Matrix(nn, nn, "u64"), Matrix(nn, nn))


def test_argument_errors():
    fb.init()
    t, small = op(), op(8)
    assert call([0], [1], [t], [t], out=False)[0] == -2                       # GrB_NULL_POINTER: out_p
    assert call([0], [1], [t], [t], nf=0)[0] == -3                            # GrB_INVALID_VALUE: nf < 1
    assert call([0], [1], [t], [t], nb=0)[0] == -3                            # nb < 1
    for lo in (2, 3):
        assert call([0], [1], [t], [t], lo=lo)[0] == -3                       # min_hops > 1
    assert call([0], [1], [(Matrix(16, 8, "u64"), None, None)], [t])[0] == -6   # GrB_DIMENSION_MISMATCH
    assert call([0], [1], [t], [small])[0] == -6
    assert call([0], [1], [t, small], [t])[0] == -6
    assert call([0], [1], [(t[0], small[1], None)], [t])[0] == -6
    assert call([16], [1], [t], [t])[0] == -4                                 # GrB_INVALID_INDEX
    assert call([0], [16], [t], [t])[0] == -4
    assert call([0], [1], [op(huge=True)], [op(huge=True)])[0] == -8          # GrB_NOT_IMPLEMENTED: host-resident operands


def test_no_pairs_do_no_device_work():
    fb.init()
    t = op()
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    info, p, nodes, nn = call([], [], [t], [t])
    assert info == 0 and p.tolist() == [0] and nn == 0
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_shortest_path_fails_loudly_without_gpu():
    fb.init()
    t = op()
    t[0].set(0, 1, 7)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    for lo, hi in ((0, 0), (1, 1), (1, (1 << 64) - 1)):
        assert call([0, 1, 2], [1, 1, 3], [t], [t, t], lo=lo, hi=hi)[0] == -7002   # GxB_GPU_ERROR
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before
    assert t[0].pending()                                                     # the queued write was not finished by the call
    with pytest.raises(fb.GrbError) as e:
        fb.shortest_path([0], [1], [t[0]], [t[0]], fwd_deltas=[t[1:]], bwd_deltas=[t[1:]])
    assert e.value.info == -7002
