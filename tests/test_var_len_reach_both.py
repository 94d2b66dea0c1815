"""B200_var_len_reach_both against the DISTINCT endpoints of the reference's DFS under Both (fdbh_var_len_trails_dfs), over
relationship tensors with pending writes of every kind, one and two types, windows min 0 / 1 x max 0 .. 4 and unbounded ones on a
small cyclic graph.  Each way a trail closes at its start is checked at k = g - 1 (excluded) and k = g (included): self-loops in the
base, deleted through dm and added through dp; reciprocal and multi-edge pairs (base pairs losing an id through me_dm); a pair shared by
two types; a triangle and a square; a hub whose only cycle joins its neighbours of rank 0 and 64; a tree; a 40-cycle.  Also more
than 1024 closure rows (with a start's rows straddling the chunk boundary, decided on either side of it) and more than 1024 starts
in one call, repeated / isolated / last-id / empty start lists, the layers
unchanged with no base downloaded, and the host mirror's C++ test."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from falkordb_b200._lib import lib, U64

pytestmark = pytest.mark.gpu
BOTH = fb.DIR_BOTH


def make_types(n, m, seed):
    """two types over n nodes with pending writes of every kind; they share pairs, and the graph has self-loops and reciprocal edges"""
    rng = np.random.default_rng(seed)
    out, nid = [], [seed * 1000000]

    def ids(k):
        a = np.arange(nid[0], nid[0] + k, dtype=np.uint64)
        nid[0] += k
        return a
    s, d = rng.integers(0, n, m), rng.integers(0, n, m)
    s[:4], d[:4] = [0, 1, 2, 3], [1, 0, 2, 3]                      # a reciprocal pair and two self-loops
    for t in range(2):
        ss, dd = (s, d) if t == 0 else (np.concatenate([s[:m // 3], rng.integers(0, n, m // 2)]),
                                        np.concatenate([d[:m // 3], rng.integers(0, n, m // 2)]))   # type 1 shares a third of the pairs
        i0 = ids(len(ss))
        T = hm.Tensor(n, ss, dd, i0)                                 # device-built base
        k = len(ss)
        rm = np.arange(0, k, 5)
        T.remove(i0[rm], ss[rm], dd[rm])                             # dm on base pairs
        T.add(ss[1:k:7], dd[1:k:7], ids(len(range(1, k, 7))))       # second ids on base pairs: multi-edge pairs in me_dp
        T.add(ss[rm[::2]], dd[rm[::2]], ids(len(rm[::2])))          # re-adds of deleted pairs
        a2, b2 = rng.integers(0, n, m // 4), rng.integers(0, n, m // 4)
        T.add(np.concatenate([a2, a2[:3], [5]]), np.concatenate([b2, b2[:3], [5]]), ids(len(a2) + 4))   # dp, pairs born multi, a self-loop
        rm2 = np.array([x for x in range(1, k, 7)[::2] if x % 5], dtype=np.int64)
        T.remove(i0[rm2], ss[rm2], dd[rm2])                          # multi-edge pairs losing a base id (me_dm)
        c = T.counts()
        assert c[0] > 0 and c[1] > 0, "test setup: dp and dm hold pending writes"
        out.append(T)
    return out


def device(types, starts, lo, hi):
    L = [t.layers() for t in types]
    n = U64(0)
    lib().GrB_Matrix_ncols(C.byref(n), L[0][0])
    R = fb.var_len_reach_both(starts, L, lo, hi)
    assert (R.nrows(), R.ncols()) == (len(starts), n.value)
    I, J, _ = R.extract_tuples()
    return set(zip(I.tolist(), J.tolist()))


def dfs(types, starts, lo, hi):
    w = hm.var_len_trails(types, starts, BOTH, lo, hi, emit_path=False, route=hm.ROUTE_BY_GET)
    row = np.repeat(np.arange(len(starts)), np.diff(w["p"]).astype(np.int64))
    return set(zip(row.tolist(), w["end"].tolist()))


def check(types, starts, lo, hi):
    got = device(types, starts, lo, hi)
    assert got == dfs(types, starts, lo, hi), (lo, hi)
    return got


@pytest.fixture(scope="module")
def graph():
    fb.init()
    return make_types(96, 200, 1)


def test_windows_and_types_equal_the_dfs(graph):
    starts = [0, 1, 2, 3, 5, 7, 7, 40, 95, 0]
    total = closed = 0
    for types in (graph[:1], graph):
        for lo in (0, 1):
            for hi in (0, 1, 2, 3, 4):
                got = check(types, starts, lo, hi)
                total += len(got)
                closed += lo == 1 and sum((i, s) in got for i, s in enumerate(starts))
    assert total > 2000 and closed > 20


def test_unbounded_on_a_small_cyclic_graph():
    fb.init()
    A = hm.Tensor(8, [0, 1, 2, 3, 4, 1, 2, 6], [1, 2, 3, 4, 0, 2, 2, 7], [0, 1, 2, 3, 4, 5, 6, 7])
    A.remove([6], [2], [2])                                      # a self-loop deleted through dm
    A.add([3, 5], [1, 6], [8, 9])
    B = hm.Tensor(8, [0, 4], [1, 2], [20, 21])
    B.add([2, 5], [5, 5], [22, 23])
    for types in ([A], [A, B]):
        for lo in (0, 1):
            got = check(types, list(range(8)) + [3], lo, None)
            assert len(got) > 20


def closes(types, s, k):
    """whether the device emits s from s at k hops (min 1), held equal to the DFS"""
    got = check(types, [s], 1, k)
    return (0, s) in got


def tensor(n, edges, first=0):
    e = np.array(edges, dtype=np.uint64).reshape(-1, 2)
    return hm.Tensor(n, e[:, 0], e[:, 1], np.arange(first, first + len(e), dtype=np.uint64))


def test_each_closure_at_its_girth():
    fb.init()
    tail = [(0, 7), (7, 8)]                                        # a path off the start, so that its rows are not empty
    T = tensor(10, tail + [(0, 0)])                                # a base self-loop: g = 1
    assert closes([T], 0, 1)
    T = tensor(10, tail + [(0, 0)])
    T.remove([2], [0], [0])                                        # ... deleted through dm
    assert not closes([T], 0, 1) and not closes([T], 0, None)
    T = tensor(10, tail)
    T.add([0], [0], [50])                                          # ... added through dp
    assert closes([T], 0, 1)
    T = tensor(10, tail + [(0, 1), (1, 0)])                        # a reciprocal pair: g = 2
    assert not closes([T], 0, 1) and closes([T], 0, 2) and closes([T], 1, 2)
    T = tensor(10, tail + [(0, 1)])
    T.add([0], [1], [50])                                          # a multi-edge pair with two live ids
    assert not closes([T], 0, 1) and closes([T], 0, 2) and closes([T], 1, 2)
    T = tensor(10, tail + [(0, 1), (0, 1), (0, 1)])                # a multi-edge pair of three base ids ...
    T.remove([3], [0], [1])                                        # ... one of them deleted through me_dm: two stay live
    assert T.counts()[5] > 0
    assert not closes([T], 0, 1) and closes([T], 0, 2)
    T = tensor(10, tail + [(0, 1), (0, 1)])                        # a multi-edge pair of two base ids ...
    T.remove([3], [0], [1])                                        # ... whose second id goes to me_dm: one stays live
    assert T.counts()[5] > 0
    assert not closes([T], 0, 2) and not closes([T], 0, None)
    A, B = tensor(10, tail + [(0, 1)]), tensor(10, [(0, 1)], 100)  # a pair shared by two types
    assert not closes([A], 0, None) and not closes([A, B], 0, 1) and closes([A, B], 0, 2)
    T = tensor(10, tail + [(0, 1), (1, 2), (2, 0)])                # a triangle: g = 3
    assert not closes([T], 0, 2) and closes([T], 0, 3) and closes([T], 2, 3)
    T = tensor(10, tail + [(0, 1), (2, 1), (2, 3), (0, 3)])        # a square with mixed directions: g = 4
    assert not closes([T], 0, 3) and closes([T], 0, 4) and closes([T], 3, 4)
    T = tensor(10, tail + [(0, 1), (2, 1), (2, 3)])
    T.add([3], [0], [60])                                          # the square closed through dp
    assert not closes([T], 0, 3) and closes([T], 0, 4)


def test_hub_whose_only_cycle_joins_ranks_0_and_64():
    fb.init()
    deg = 72
    edges = [(0, c) for c in range(1, deg + 1)] + [(1, 65)]      # neighbours 1 .. 72 have ranks 0 .. 71; 1 and 65 differ in bit 6
    T = tensor(deg + 1, edges)
    assert not closes([T], 0, 2) and closes([T], 0, 3)
    T = tensor(deg + 1, edges[:-1])
    T.add([65], [1], [500])                                        # the same chord as a pending insert, reversed
    assert not closes([T], 0, 2) and closes([T], 0, 3)
    T = tensor(deg + 1, edges[:-1] + [(1, 2)])                   # ranks 0 and 1 (bit 0) as a control
    assert closes([T], 0, 3)


def test_tree_and_a_40_cycle():
    fb.init()
    tree = [(0, 1), (0, 2), (1, 3), (1, 4), (2, 5), (5, 6), (6, 7)]
    T = tensor(8, tree)
    for s in range(8):
        assert not closes([T], s, None)
    ring = [(v, (v + 1) % 40) for v in range(40)]
    T = tensor(41, ring + [(0, 40)])
    assert not closes([T], 0, 39) and closes([T], 0, 40) and closes([T], 0, None) and closes([T], 17, None)
    assert not closes([T], 40, None)


@pytest.mark.parametrize("chord", [(0, 1), (0, 8)])
def test_more_than_1024_closure_rows_and_starts(chord):
    fb.init()
    # 300 stars: star 0 has 8 leaves (3 closure rows), the others 16 (4 rows), 1,199 rows in all, so star 256's rows are 1,023 ..
    # 1,026 and straddle the first chunk's end.  Every third star has a chord between two leaves (g = 3), every fifth one a leaf
    # path of two edges between leaves (g = 4), and star 256 a chord between the leaves of ranks `chord`: ranks 0 and 1 differ in
    # bit 0 (row 1,023: decided in the first chunk, its rows of the second chunk are not seeded), 0 and 8 in bit 3 (row 1,026:
    # decided in the second chunk).  The rest have no cycle.
    hubs, edges, rows, n = [], [], [], 0
    for h in range(300):
        c, nl = n, 8 if h == 0 else 16
        leaves = list(range(c + 1, c + 1 + nl))
        edges += [(c, x) if x % 2 else (x, c) for x in leaves]
        if h % 3 == 0:
            edges.append((leaves[h % nl], leaves[(h * 7 + 3) % nl]))   # 6h + 3 is odd: two distinct leaves
        elif h % 5 == 0:
            edges += [(leaves[0], c + 1 + nl), (c + 1 + nl, leaves[9])]
        elif h == 256:
            edges.append((leaves[chord[0]], leaves[chord[1]]))
        hubs.append(c)
        rows.append(int(nl - 1).bit_length())
        n = c + 2 + nl
    first = np.cumsum([0] + rows)
    assert first[256] < 1024 < first[257], "test setup: star 256's rows straddle the chunk boundary"
    T = tensor(n + 1, edges)
    for k in (3, 4):
        got = check([T], hubs, 1, k)
        closed = {hubs[i] for i, v in got if v == hubs[i]}
        assert closed == {hubs[h] for h in range(300) if h % 3 == 0 or h == 256 or (k >= 4 and h % 5 == 0)}
    many = (hubs * 4)[:1100] + [n, n - 1]                          # more than 1024 starts: the reach takes its row-wise path
    check([T], many, 1, 4)
    check([T], many, 0, 3)


def test_start_lists(graph):
    for starts in ([], [60], [60, 60], [95, 94, 93], [4] * 5):
        for lo, hi in ((1, 3), (0, 2), (1, 1)):
            check(graph[:1], starts, lo, hi)
    R = fb.var_len_reach_both([], [t.layers() for t in graph], 1, 3)
    assert (R.nrows(), R.nvals()) == (0, 0)


def test_layers_unchanged_and_no_base_download():
    fb.init()
    types = make_types(2000, 8000, 3)                                # bases built on the device: no host form until tuples() reads them
    L = [t.layers() for t in types]
    starts = list(range(0, 2000, 40))
    fb.reset_stats()
    d0 = fb.get_stat("d2h_bytes")
    R = fb.var_len_reach_both(starts, L, 1, 4)                       # first: nothing has read the layers yet
    moved = fb.get_stat("d2h_bytes") - d0
    base = sum(len(t.tuples()[0][0]) for t in types) * 12            # what downloading the two bases would move (ids and values)
    assert moved <= 4096 < base, (moved, base)                       # a few words per call and level; the result stays on the device
    assert R.nvals() > 1000
    before = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    R2 = fb.var_len_reach_both(starts, L, 1, 4)
    after = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    assert before == after
    assert R2.tuple_set() == R.tuple_set()


def test_host_mirror_var_len_reach_both_matches_trails():
    fb.init()
    L = hm.host()
    assert L.fdbh_run_test(b"var_len_reach_both_matches_trails") == 0, L.fdbh_last_message().decode()
