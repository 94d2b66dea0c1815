"""B200_all_shortest_paths (through the host mirror's all_shortest_paths: a counting call, then windows) against the reference's
route (all_shortest_paths_by_iter: expand_row over TypesAdjacency), edge list for edge list and node list for node list, in order.
Tensors carry pending writes of every kind (dp, dm, MULTI_EDGE pairs, deleted multi-edge ids).  Covered: 1-3 types, named subsets
with missing types, untyped patterns, Out and Both, cycles including a self-loop on src, unreachable and beyond-max_hops pairs,
more than 1,024 pairs, levels cut into pieces, draining in small windows, and, on tensors written only on the device, the layers
unchanged with only the outputs and a few words per level moved to the host.  The reference route is also held to the Python
transcription of expand_row."""
import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from test_all_shortest_paths_abi import Graph, expand_row
from test_shortest_path import device_built, effective, make_graph

pytestmark = pytest.mark.gpu
INF = None


def both_routes(types, named, srcs, dsts, directed, hi, window=1 << 22):
    dev = hm.all_shortest_paths(types, named, srcs, dsts, directed, hi, route=hm.ASP_DEVICE, window=window)
    ref = hm.all_shortest_paths(types, named, srcs, dsts, directed, hi, route=hm.ASP_BY_ITER)
    assert dev == ref, (len(named), directed, hi)
    return dev


def named_lists(types):
    out = [[]] + [[t] for t in types]
    if len(types) > 1:
        out.append([types[-1], types[0]])
        out.append(list(types) + [None])                           # a missing type, dropped
    out.append([None])                                              # every named type missing
    return out


@pytest.fixture(scope="module")
def graphs():
    fb.init()
    return {k: make_graph(48, 80, k, 40 + k) for k in (1, 2, 3)}


@pytest.mark.parametrize("ntypes", [1, 2, 3])
def test_device_equals_reference_route(graphs, ntypes):
    types, _ = graphs[ntypes]
    rng = np.random.default_rng(ntypes)
    srcs = [int(x) for x in rng.integers(0, 48, 40)] + [5, 2, 0, 47]
    dsts = [int(x) for x in rng.integers(0, 48, 40)] + [5, 2, 0, 46]
    paths = 0
    for named in named_lists(types):
        for directed in (True, False):
            for hi in (1, 2, 3, INF):
                got = both_routes(types, named, srcs, dsts, directed, hi)
                paths += sum(len(x) for x in got)
    assert paths > 300


def test_reference_route_equals_the_transcription(graphs):
    for ntypes in (1, 3):
        types, _ = graphs[ntypes]
        rels = effective(types, 48)
        rng = np.random.default_rng(7 + ntypes)
        srcs = [int(x) for x in rng.integers(0, 48, 25)] + [5, 2]
        dsts = [int(x) for x in rng.integers(0, 48, 25)] + [5, 2]
        for pick in ([], [ntypes - 1, 0]):
            named = [types[t] for t in pick]
            g = Graph(rels, [f"T{t}" for t in (pick or range(ntypes))])
            for directed in (True, False):
                for hi in (INF, 2):
                    got = hm.all_shortest_paths(types, named, srcs, dsts, directed, hi, route=hm.ASP_BY_ITER)
                    assert got == [expand_row(g, not directed, hi, s, d) for s, d in zip(srcs, dsts)]


def test_cycles_self_loops_and_unreachable_pairs():
    fb.init()
    # 0 has two self-loops (one type each) and a 2-cycle with 1; 2 -> 3 -> 4 -> 2 is a 3-cycle; 5 is isolated; 6 -> 7 is one way
    R = hm.Tensor(8, [0, 0, 1, 2, 3, 4, 6], [0, 1, 0, 3, 4, 2, 7], [10, 11, 12, 13, 14, 15, 16])
    S = hm.Tensor(8, [0, 3], [0, 4], [20, 21])                       # a parallel 3 -> 4 in another type
    srcs, dsts = [0, 1, 2, 2, 5, 7, 6, 2], [0, 1, 2, 4, 5, 6, 7, 0]
    for directed in (True, False):
        for hi in (1, 2, INF):
            got = both_routes([R, S], [], srcs, dsts, directed, hi)
            assert [p[0] for p in got[0]] == [[20], [10]]           # the self-loops, the last-listed predecessor first
            assert got[4] == [] and got[7] == []
            if directed:
                assert got[5] == []
    R.remove([10], [0], [0])                                          # a pending delete of one self-loop
    assert [p[0] for p in both_routes([R, S], [], [0], [0], True, INF)[0]] == [[20]]


def test_more_than_one_slice_and_pieces(graphs):
    types, _ = graphs[2]
    rng = np.random.default_rng(9)
    srcs = [int(x) for x in rng.integers(0, 48, 1100)]
    dsts = [int(x) for x in rng.integers(0, 48, 1100)]
    for directed in (True, False):
        both_routes(types, [], srcs, dsts, directed, INF)
    try:
        for budget in (1, 7):                                        # every front entry its own piece, and a few per piece
            fb.set_option("shortest_path_budget", budget)
            for named in ([], types[:1]):
                for directed in (True, False):
                    both_routes(types, named, srcs[:200], dsts[:200], directed, INF)
                    both_routes(types, named, srcs[:40], dsts[:40], directed, 2)
    finally:
        fb.set_option("shortest_path_budget", 0)


def test_draining_in_small_windows(graphs):
    types, _ = graphs[3]
    rng = np.random.default_rng(3)
    srcs = [int(x) for x in rng.integers(0, 48, 60)]
    dsts = [int(x) for x in rng.integers(0, 48, 60)]
    for directed in (True, False):
        whole = hm.all_shortest_paths(types, [], srcs, dsts, directed, INF, route=hm.ASP_DEVICE)
        for window in (1, 3, 10):
            assert hm.all_shortest_paths(types, [], srcs, dsts, directed, INF, route=hm.ASP_DEVICE, window=window) == whole
        # one call from given ranks on: the rest of each pair, pairs filled in order until a path no longer fits
        full = fb.all_shortest_paths(srcs, dsts, [t.layers() for t in types], fb.DIR_OUT if directed else fb.DIR_BOTH)
        first = [min(int(c), 2) for c in full["count"]]
        part = fb.all_shortest_paths(srcs, dsts, [t.layers() for t in types], fb.DIR_OUT if directed else fb.DIR_BOTH, first=first,
                                     edge_capacity=25)
        e, k, stop = 0, 0, False
        for i in range(len(srcs)):
            c, ln = int(full["count"][i]), int(full["len"][i])
            w = int(part["p"][i + 1] - part["p"][i])
            want = 0 if stop else min(c - first[i], (25 - e) // ln if ln else 0)
            stop = stop or want < c - first[i]
            assert w == want, i
            for r in range(first[i], first[i] + w):
                edges = [x for x in whole[i][r][0]]
                assert part["edges"][e:e + ln].tolist() == edges
                assert part["nodes"][e + k:e + k + ln + 1].tolist() == whole[i][r][1]
                e += ln
                k += 1


def test_layers_unchanged_and_no_base_download():
    fb.init()
    types = device_built(3000, 9000, 2, 4)                           # nothing reads the layers before the measured call
    srcs, dsts = list(range(0, 3000, 30)), list(range(7, 3000, 30)) + [0]
    srcs.append(0)
    L = [t.layers() for t in types]
    fb.reset_stats()
    got = fb.all_shortest_paths(srcs, dsts, L, fb.DIR_BOTH, max_hops=6)
    moved = fb.get_stat("d2h_bytes")
    assert (got["count"] > 0).sum() > 10
    out = 2 * 12 * len(srcs) + 12 * len(got["edges"]) + 4 * len(got["nodes"])   # a counting call, then the filling one
    base = sum(len(t.tuples()[0][0]) for t in types) * 12           # what downloading the two bases would move (ids and values)
    assert moved <= out + 64 * 6 * 4 < base, (moved, out, base)      # the outputs and a few words per level
    before = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    again = fb.all_shortest_paths(srcs, dsts, L, fb.DIR_BOTH, max_hops=6)
    after = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    assert before == after
    assert all(np.array_equal(got[k], again[k]) for k in got)
