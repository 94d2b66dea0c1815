"""B200_var_len_trails against the reference's DFS (fdbh_var_len_trails_dfs: VarLenIterT over TypesAdjacency), list for list in
start, end, hops, edges and nodes, over relationship tensors with pending writes: dp / dm on base pairs, multi-edge pairs gaining
and losing ids in me_dp / me_dm, reciprocal edges and self-loops, and two types sharing a pair.  Out / In / Both, hop windows
including 0 and unbounded, fixed destinations, destination labels with pending label writes or a missing label, repeated,
isolated and empty start lists; a hub whose expansion takes several grid sweeps, a 64-edge path, GrB_INSUFFICIENT_SPACE on both
capacities, and the layers untouched with no base downloaded."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from falkordb_b200._lib import lib, P, U64
from falkordb_b200.grb import TensorLayers

pytestmark = pytest.mark.gpu
U64MAX = (1 << 64) - 1
OUT, IN, BOTH = fb.DIR_OUT, fb.DIR_IN, fb.DIR_BOTH


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


def same(a, b):
    for k in ("p", "end", "hops", "edges", "nodes"):
        assert np.array_equal(a[k].astype(np.uint64), b[k].astype(np.uint64)), k


def both_routes(types, starts, dir, lo, hi, dests=None, labels=(), emit_path=True):
    want = hm.var_len_trails(types, starts, dir, lo, hi, dests, labels, emit_path, route=hm.ROUTE_BY_GET)
    got = hm.var_len_trails(types, starts, dir, lo, hi, dests, labels, emit_path, route=hm.ROUTE_DEVICE)
    same(got, want)
    return want


@pytest.fixture(scope="module")
def graph():
    fb.init()
    return make_types(96, 200, 1)


@pytest.fixture(scope="module")
def small():
    """two types over 6 nodes, small enough for unbounded windows: a 5-cycle, a reciprocal edge, a self-loop, a multi-edge pair, a
    pair shared by both types; pending deletes and inserts in both"""
    fb.init()
    A = hm.Tensor(6, [0, 1, 2, 3, 4, 1, 2, 3], [1, 2, 3, 4, 0, 2, 2, 1], [0, 1, 2, 3, 4, 5, 6, 7])
    A.remove([7], [3], [1])
    A.add([3, 1, 5], [1, 2, 0], [8, 9, 10])                     # a re-add, a third id on (1, 2), a new edge
    A.remove([5], [1], [2])                                     # (1, 2) loses a base id
    B = hm.Tensor(6, [0, 4], [1, 2], [20, 21])
    B.add([2, 5], [5, 5], [22, 23])
    B.remove([21], [4], [2])
    return [A, B]


WINDOWS = [(0, 0), (0, 1), (1, 1), (1, 3), (2, 2), (2, 4), (3, 5)]


@pytest.mark.parametrize("dir", [OUT, IN, BOTH])
def test_windows_and_types_equal_the_dfs(graph, dir):
    starts = [0, 1, 2, 3, 5, 7, 7, 40, 95, 0]
    total = 0
    for types in (graph[:1], graph):
        for lo, hi in WINDOWS:
            if dir == BOTH and hi == 5:
                hi = 4
            total += len(both_routes(types, starts, dir, lo, hi)["end"])
    assert total > 1000


@pytest.mark.parametrize("dir", [OUT, IN, BOTH])
def test_unbounded_on_a_small_cyclic_graph(small, dir):
    for lo in (0, 1, 2):
        w = both_routes(small, list(range(6)) + [3], dir, lo, None)
        assert len(w["end"]) > 10


@pytest.mark.parametrize("dir", [OUT, IN, BOTH])
def test_fixed_destinations_and_labels(graph, dir):
    n = 96
    starts = [0, 1, 2, 3, 5, 9, 9, 50]
    dests = [1, -1, 2, 3, -1, 9, 10, -1]
    la, lb = hm.VersionedMatrix(n), hm.VersionedMatrix(n)
    for v in range(0, n, 2):
        la.set(v, v)
    for v in range(0, n, 3):
        lb.set(v, v)
    la.set_all(list(range(1, n, 6)), list(range(1, n, 6)))       # pending label adds
    for v in range(0, n, 12):
        la.remove(v, v)                                            # pending label deletes
    for labels in ((), (la,), (la, lb), (la, None)):
        for lo, hi in ((0, 2), (1, 3), (2, 4)):
            both_routes(graph, starts, dir, lo, hi, None, labels)
            both_routes(graph, starts, dir, lo, hi, dests, labels)
            if labels and labels[-1] is None:
                assert len(hm.var_len_trails(graph, starts, dir, lo, hi, None, labels)["end"]) == 0


def test_start_lists_and_count_modes(graph):
    for starts in ([], [60], [60, 60], [95, 94, 93], [4] * 5):
        for dir in (OUT, IN, BOTH):
            both_routes(graph, starts, dir, 1, 3)
            both_routes(graph, starts, dir, 0, 2, emit_path=False)
    L = [x for x in (graph[0].layers(), graph[1].layers())]
    full = fb.var_len_trails([0, 1, 2], L, OUT, 1, 3)
    cnt = fb.var_len_trails([0, 1, 2], L, OUT, 1, 3, mode="count")
    ends = fb.var_len_trails([0, 1, 2], L, OUT, 1, 3, mode="ends")
    assert np.array_equal(cnt["p"], full["p"]) and cnt["npath"] == full["npath"] == int(full["hops"].sum())
    assert np.array_equal(ends["end"], full["end"]) and np.array_equal(ends["hops"], full["hops"])


def test_hub_over_several_grid_sweeps():
    fb.init()
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    N = 2 * sms * 4096 + 7
    leaves = np.arange(1, N + 1, dtype=np.uint64)
    back = leaves[::9973]
    src = np.concatenate([np.zeros(N, np.uint64), back, [0]])
    dst = np.concatenate([leaves, np.zeros(len(back), np.uint64), [5]])          # 0 -> 5 twice: a multi-edge pair
    T = hm.Tensor(N + 1, src, dst, np.arange(len(src), dtype=np.uint64))
    T.add([0, 7], [7, 0], [10 ** 8, 10 ** 8 + 1])
    T.remove([3], [0], [4])                                                        # edge id 3 is 0 -> 4
    for dir, lo, hi in ((OUT, 1, 2), (IN, 1, 2), (BOTH, 1, 2), (OUT, 2, 2)):
        w = both_routes([T], [0, back[1], 0], dir, lo, hi, emit_path=(hi == 2))
        assert len(w["end"]) > (N if dir != IN else 100)


def test_64_edge_path_unbounded():
    fb.init()
    src, dst = np.arange(64, dtype=np.uint64), np.arange(1, 65, dtype=np.uint64)
    T = hm.Tensor(65, src, dst, np.arange(64, dtype=np.uint64) + 100)
    for dir, s in ((OUT, 0), (IN, 64), (BOTH, 0), (BOTH, 32)):
        w = both_routes([T], [s], dir, 1, None)
        assert len(w["end"]) == 64
        assert w["hops"].max() == (32 if s == 32 else 64)


def raw(starts, layers, dir, lo, hi, cap, pcap, tree=U64MAX):
    starts = np.ascontiguousarray(starts, dtype=np.uint64)
    ls = (TensorLayers * len(layers))()
    for k, t in enumerate(layers):
        for name, x in zip(("m", "dp", "dm", "mt", "mt_dp", "mt_dm", "me", "me_dp", "me_dm"), t):
            setattr(ls[k], name, x)
    pp = np.full(len(starts) + 1, 77, np.uint64)
    oe, oh = np.full(max(cap, 1), 77, np.uint32), np.full(max(cap, 1), 77, np.uint32)
    pe, pn = np.full(max(pcap, 1), 77, np.uint64), np.full(max(pcap + cap, 1), 77, np.uint32)
    nv, npth = U64(0), U64(0)
    info = lib().B200_var_len_trails(starts.ctypes.data, None, len(starts), ls, len(layers), dir, lo, hi, None, None, None, 0, tree,
                                     pp.ctypes.data, oe.ctypes.data, oh.ctypes.data, cap, pe.ctypes.data, pn.ctypes.data, pcap,
                                     C.byref(nv), C.byref(npth))
    return info, pp, oe, oh, pe, pn, nv.value, npth.value


def test_insufficient_space_writes_nothing_and_a_retry_is_equal(graph):
    L = [t.layers() for t in graph]
    starts = [0, 1, 2, 3, 40]
    full = fb.var_len_trails(starts, L, BOTH, 1, 3)
    nout, npath = full["nout"], full["npath"]
    assert nout > 100
    for cap, pcap in ((nout - 1, npath), (nout, npath - 1), (0, 0)):
        info, pp, oe, oh, pe, pn, nv, np_ = raw(starts, L, BOTH, 1, 3, cap, pcap)
        assert info == -103 and nv == nout and np_ == npath and np.array_equal(pp, full["p"])
        assert (oe == 77).all() and (oh == 77).all() and (pe == 77).all() and (pn == 77).all()
    stored = int(fb.var_len_trails(starts, L, BOTH, 1, 2, mode="count")["nout"])   # levels 1-2 of *1..3: the trails of 1 and 2 hops
    info, pp, oe, oh, pe, pn, nv, np_ = raw(starts, L, BOTH, 1, 3, nout, npath, tree=stored - 1)
    assert info == -103 and nv == U64MAX and np_ == U64MAX
    assert (pp == 77).all() and (oe == 77).all() and (pe == 77).all()
    info, pp, oe, oh, pe, pn, nv, np_ = raw(starts, L, BOTH, 1, 3, nout, npath, tree=stored)
    assert info == 0 and nv == nout
    assert np.array_equal(pp, full["p"]) and np.array_equal(oe[:nout], full["end"]) and np.array_equal(pe[:npath], full["edges"])
    assert np.array_equal(pn[:npath + nout], full["nodes"])


def test_layers_unchanged_and_no_base_download():
    fb.init()
    types = make_types(2000, 8000, 3)                                # bases built on the device: no host form
    L = [t.layers() for t in types]
    starts = list(range(0, 2000, 40))
    fb.reset_stats()
    d0 = fb.get_stat("d2h_bytes")
    r = fb.var_len_trails(starts, L, OUT, 1, 3)
    moved = fb.get_stat("d2h_bytes") - d0
    out = 8 * (len(starts) + 1) + 4 * 2 * r["nout"] + 12 * r["npath"] + 4 * r["nout"]
    assert moved <= 2 * out + 4096, (moved, out)                     # the outputs, twice for the count call, plus a few words a level
    before = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    fb.var_len_trails(starts, L, BOTH, 0, 2)
    after = [[(len(a[0]), np.sum(a[0]), np.sum(a[1])) for a in t.tuples()] for t in types]
    assert before == after
