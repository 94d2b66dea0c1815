"""B200_shortest_path (through the host mirror's shortest_path: the device BFS, then B200_expand_edges for the ids) against the
reference's route (shortest_path_by_iter: NeighborIter's BFS and Tensor::get), row for row: nodes, relationship ids and Nulls.
Relationship tensors carry pending writes of every kind; the adjacency VersionedMatrix carries pending inserts and deletes.  Covered:
1-3 types, named subsets with missing types, untyped patterns, directed and undirected, min_hops 0 / 1 with max_hops 0 .. 3 and
unbounded, src == dst rows, the flow test's 5-node graph, tie-heavy graphs (layered complete bipartite, grids) and equal front sizes,
batches within one slice and over 1,024 pairs, rounds cut into many pieces, an adjacency without relationship types, and the
layers unchanged with only the paths moved to the host on tensors built and written on the device only.  Both routes are also held
to the Python transcription of bfs_shortest_path on 1,000 small random multigraphs."""
import json

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from test_shortest_path_abi import GOLDEN, bfs_shortest_path, sides

pytestmark = pytest.mark.gpu
INF = None
WINDOWS = [(lo, hi) for lo in (0, 1) for hi in (0, 1, 2, 3, INF)]


def make_graph(n, m, ntypes, seed):
    """ntypes Tensors over n nodes with pending writes of every kind (self-loops, reciprocal pairs, multi-edges, deletes and
    re-adds), and the adjacency VersionedMatrix of their effective pairs, part of it pending"""
    rng = np.random.default_rng(seed)
    out, nid = [], [seed * 1000000]

    def ids(k):
        a = np.arange(nid[0], nid[0] + k, dtype=np.uint64)
        nid[0] += k
        return a
    for t in range(ntypes):
        s, d = rng.integers(0, n, m), rng.integers(0, n, m)
        s[:4], d[:4] = [0, 1, 2, 3], [1, 0, 2, 3]
        i0 = ids(m)
        T = hm.Tensor(n, s, d, i0)
        rm = np.arange(0, m, 5)
        T.remove(i0[rm], s[rm], d[rm])
        T.add(s[1:m:7], d[1:m:7], ids(len(range(1, m, 7))))
        T.add(s[rm[::2]], d[rm[::2]], ids(len(rm[::2])))
        a2, b2 = rng.integers(0, n, m // 4), rng.integers(0, n, m // 4)
        T.add(np.concatenate([a2, [5]]), np.concatenate([b2, [5]]), ids(len(a2) + 1))
        out.append(T)
    adj = hm.VersionedMatrix(n)
    pairs = effective(out, n)
    keys = sorted({(u, v) for rels in pairs.values() for u, v, _ in rels})
    half = len(keys) // 2
    if keys:
        r, c = zip(*keys[:half]) if half else ((), ())
        if half:
            adj.set_all(r, c)
        for u, v in keys[half:]:
            adj.set(u, v)
    return out, adj


def effective(types, n):
    """{type index: [(u, v, id)]}: every live relationship, read through the reference's Tensor::get route"""
    rels = {}
    for k, T in enumerate(types):
        p, node, edge, _, _ = hm.expand_edges([T], list(range(n)), fb.DIR_OUT, fb.EDGES_ALL)
        rels[f"T{k}"] = [(u, int(node[q]), int(edge[q])) for u in range(n) for q in range(int(p[u]), int(p[u + 1]))]
    return rels


def both_routes(adj, types, named, srcs, dsts, directed, lo, hi):
    dev = hm.shortest_path(adj, types, named, srcs, dsts, directed, lo, hi, route=hm.SP_DEVICE)
    ref = hm.shortest_path(adj, types, named, srcs, dsts, directed, lo, hi, route=hm.SP_BY_ITER)
    assert dev == ref, (named, directed, lo, hi)
    return dev


def named_lists(types):
    ks = list(range(len(types)))
    out = [[]]
    for k in ks:
        out.append([types[k]])
    if len(types) > 1:
        out.append([types[-1], types[0]])
        out.append(list(types) + [None])                           # a missing type, dropped
    out.append([None])                                              # every named type missing
    return out


@pytest.fixture(scope="module")
def graphs():
    fb.init()
    return {k: make_graph(64, 90, k, 10 + k) for k in (1, 2, 3)}


@pytest.mark.parametrize("ntypes", [1, 2, 3])
def test_device_equals_reference_route(graphs, ntypes):
    types, adj = graphs[ntypes]
    rng = np.random.default_rng(ntypes)
    srcs = [int(x) for x in rng.integers(0, 64, 40)] + [7, 0]
    dsts = [int(x) for x in rng.integers(0, 64, 40)] + [7, 1]
    found = 0
    for named in named_lists(types):
        for directed in (True, False):
            for lo, hi in WINDOWS:
                got = both_routes(adj, types, named, srcs, dsts, directed, lo, hi)
                found += sum(x is not None and len(x[0]) > 1 for x in got)
    assert found > 200


def test_reference_route_equals_the_transcription(graphs):
    types, adj = graphs[2]
    rel = effective(types, 64)
    names = {id(T): f"T{k}" for k, T in enumerate(types)}
    rng = np.random.default_rng(5)
    srcs, dsts = [int(x) for x in rng.integers(0, 64, 30)], [int(x) for x in rng.integers(0, 64, 30)]
    for named in ([], [types[1]], [types[1], types[0]]):
        for directed in (True, False):
            fwd, bwd = sides(64, rel, [names[id(t)] for t in named], directed)
            for lo, hi in ((1, INF), (0, 2)):
                got = hm.shortest_path(adj, types, named, srcs, dsts, directed, lo, hi, route=hm.SP_BY_ITER)
                want = [bfs_shortest_path(fwd, bwd, s, d, hi, lo) for s, d in zip(srcs, dsts)]
                assert [None if x is None else x[0] for x in got] == want


def test_flow_goldens_on_the_device():
    fb.init()
    g = json.load(open(GOLDEN))
    tensors = {}
    for name, rels in g["types"].items():
        s, d, i = zip(*rels)
        tensors[name] = hm.Tensor(g["n"], s, d, i)
    all_types = list(tensors.values())
    adj = hm.VersionedMatrix(g["n"])
    r, c = zip(*sorted({(u, v) for rels in g["types"].values() for u, v, _ in rels}))
    adj.set_all(r, c)
    ids = {(u, v): i for rels in g["types"].values() for u, v, i in rels}
    for case in g["cases"]:
        named = [tensors.get(t) for t in case["named"]]
        got = both_routes(adj, all_types, named, case["src"], case["dst"], case["directed"], case["min_hops"], case["max_hops"])
        assert [None if x is None else x[0] for x in got] == case["nodes"], case["name"]
        for x in got:
            if x is not None:
                assert x[1] == [ids[(u, v)] for u, v in zip(x[0], x[0][1:])]


def test_ties_grids_and_equal_fronts():
    fb.init()
    # layered complete bipartite: 1 - 4 - 4 - 4 - 1, every route of equal length; and a 12 x 12 grid with both directions
    layers = [[0], [1, 2, 3, 4], [5, 6, 7, 8], [9, 10, 11, 12], [13]]
    es = [(u, v) for a, b in zip(layers, layers[1:]) for u in a for v in b]
    w = 12
    grid = [(r * w + c, r * w + c + 1) for r in range(w) for c in range(w - 1)] + [(r * w + c, (r + 1) * w + c) for r in range(w - 1) for c in range(w)]
    for edges, n, pairs in ((es, 14, [(0, 13), (1, 12), (5, 8), (13, 0), (2, 3)]),
                            (grid, w * w, [(0, w * w - 1), (w - 1, (w - 1) * w), (5, 77), (w * w - 1, 0), (13, 14)])):
        s, d = zip(*edges)
        T = hm.Tensor(n, s, d, np.arange(len(edges)))
        adj = hm.VersionedMatrix(n)
        adj.set_all(s, d)
        srcs, dsts = zip(*pairs)
        for named in ([], [T]):
            for directed in (True, False):
                for lo, hi in ((1, INF), (0, 3), (1, 6)):
                    both_routes(adj, [T], named, srcs, dsts, directed, lo, hi)


def test_batches_over_one_slice_and_many_pieces(graphs):
    types, adj = graphs[2]
    rng = np.random.default_rng(9)
    srcs = [int(x) for x in rng.integers(0, 64, 1100)]
    dsts = [int(x) for x in rng.integers(0, 64, 1100)]
    for named in ([], types):
        for directed in (True, False):
            both_routes(adj, types, named, srcs, dsts, directed, 1, INF)
    try:
        for budget in (1, 7):                                        # every front node its own piece, and a few per piece
            fb.set_option("shortest_path_budget", budget)
            for named in ([], types[:1], types):
                for directed in (True, False):
                    both_routes(adj, types, named, srcs[:300], dsts[:300], directed, 1, INF)
                    both_routes(adj, types, named, srcs[:40], dsts[:40], directed, 0, 2)
    finally:
        fb.set_option("shortest_path_budget", 0)


def test_adjacency_without_relationship_types():
    """untyped and directed over an adjacency with no relationship type: the backward side walks nothing, yet the forward side
    still meets dst (at depth 0 on the backward side)"""
    fb.init()
    adj = hm.VersionedMatrix(6)
    adj.set_all([0, 1, 2, 4], [1, 2, 3, 4])
    adj.remove(2, 3)
    srcs, dsts = [0, 1, 0, 4, 3, 5], [1, 2, 2, 4, 3, 0]
    for directed in (True, False):
        for lo, hi in ((1, INF), (0, INF), (1, 1)):
            got = both_routes(adj, [], [], srcs, dsts, directed, lo, hi)
            assert got[0] == ([0, 1], [])


def test_reference_route_equals_the_transcription_on_many_graphs():
    """the typed C++ reference route (its forward layers and matrix_t sides, pending writes of every kind) and the device route,
    against the Python transcription on 1,000 small random multigraphs"""
    fb.init()
    rng = np.random.default_rng(77)
    for g in range(1000):
        n = int(rng.integers(6, 20))
        ntypes = int(rng.integers(1, 4))
        types, adj = make_graph(n, int(rng.integers(5, 3 * n)), ntypes, 100 + g)
        rel = effective(types, n)
        pick = [k for k in range(ntypes) if rng.random() < 0.6]
        named = [types[k] for k in pick]
        directed = bool(g % 2)
        fwd, bwd = sides(n, rel, [f"T{k}" for k in pick], directed)
        srcs, dsts = [int(x) for x in rng.integers(0, n, 6)], [int(x) for x in rng.integers(0, n, 6)]
        lo, hi = [(1, INF), (0, 2), (1, 1), (1, 3)][g % 4]
        got = both_routes(adj, types, named, srcs, dsts, directed, lo, hi)
        want = [bfs_shortest_path(fwd, bwd, s, d, hi, lo) for s, d in zip(srcs, dsts)]
        assert [None if x is None else x[0] for x in got] == want, (g, pick, directed, lo, hi)


def device_built(n, m, ntypes, seed):
    """Tensors whose bases and pending writes were made on the device only (bulk load, then the device write plans): no layer has
    a host form until something reads it"""
    rng = np.random.default_rng(seed)
    out, nid = [], seed * 1000000
    for t in range(ntypes):
        s, d = rng.integers(0, n, m).astype(np.uint64), rng.integers(0, n, m).astype(np.uint64)
        ids = np.arange(nid, nid + m, dtype=np.uint64)
        nid += m
        T = hm.Tensor(n, s, d, ids)
        rm = np.arange(0, m, 5)
        T.remove(ids[rm], s[rm], d[rm], route=hm.WRITE_DEVICE)
        k = m // 4
        T.add(rng.integers(0, n, k).astype(np.uint64), rng.integers(0, n, k).astype(np.uint64), np.arange(nid, nid + k, dtype=np.uint64),
              route=hm.WRITE_DEVICE)
        nid += k
        c = T.counts()
        assert c[0] > 0 and c[1] > 0, "test setup: dp and dm hold pending writes"
        out.append(T)
    return out


def test_layers_unchanged_and_no_base_download():
    fb.init()
    types = device_built(3000, 9000, 2, 4)                           # nothing reads the layers before the measured call
    srcs, dsts = list(range(0, 3000, 30)), list(range(7, 3000, 30))
    L = [t.layers() for t in types]
    fwd = [(l[0], l[1], l[2]) for l in L]
    bwd = [(l[3], l[4], l[5]) for l in L]
    fb.reset_stats()
    got = fb.shortest_path(srcs, dsts, [x[0] for x in fwd], [x[0] for x in bwd], 1, None, [x[1:] for x in fwd], [x[1:] for x in bwd])
    moved = fb.get_stat("d2h_bytes")
    nodes = sum(len(x) for x in got if x is not None)
    assert sum(x is not None for x in got) > 10
    base = sum(len(t.tuples()[0][0]) for t in types) * 12           # what downloading the two bases would move (ids and values)
    assert moved <= 8 * len(srcs) + 4 * nodes < base, (moved, base)  # the path lengths and the path nodes, nothing else
    before = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    again = fb.shortest_path(srcs, dsts, [x[0] for x in fwd], [x[0] for x in bwd], 1, None, [x[1:] for x in fwd], [x[1:] for x in bwd])
    after = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    assert before == after
    assert all((a is None and b is None) or (a is not None and b is not None and np.array_equal(a, b)) for a, b in zip(got, again))
