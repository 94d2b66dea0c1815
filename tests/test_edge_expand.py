"""B200_expand_edges: the relationship ids of named-edge, incoming and bidirectional hops, and of ExpandInto's pair probes, over
relationship tensors with pending writes.  Every case is compared, array for array, with a numpy model over the tensor's layers
(Tensor::eff_get per type, MULTI_EDGE expanded through (me \\ me_dm) u me_dp) and with the route the call replaces: the host
mirror's expand_row / ExpandInto restatement over Tensor::get (expand_edges_by_get / expand_into_by_get)."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200._lib import lib, check, U64
from falkordb_b200 import host_mirror as hm
from falkordb_b200.grb import Matrix
from falkordb_b200.host_mirror import Tensor

pytestmark = pytest.mark.gpu
MULTI = (1 << 64) - 1
DIRS = (fb.DIR_OUT, fb.DIR_IN, fb.DIR_BOTH)
MODES = (fb.EDGES_ALL, fb.EDGES_FIRST)
N = 30_000
HUB = 7


def via_host(tensors, src, dir, mode, targets=None, route=1):
    """route 0: B200_expand_edges through the host mirror, 1: Tensor::get per pair, 2: bind_edge's route"""
    return hm.expand_edges(tensors, src, dir, mode, targets, route)


def tuples(h, valued):
    if h is None:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    nv = U64()
    check(lib().GrB_Matrix_nvals(C.byref(nv), h))
    k = nv.value
    I, J = np.zeros(max(k, 1), np.uint64), np.zeros(max(k, 1), np.uint64)
    X = np.zeros(max(k, 1), np.uint64 if valued else np.bool_)
    n2 = U64(k)
    f = lib().GrB_Matrix_extractTuples_UINT64 if valued else lib().GrB_Matrix_extractTuples_BOOL
    check(f(I.ctypes.data, J.ctypes.data, X.ctypes.data, C.byref(n2), h))
    return I[:k], J[:k], X[:k]


class Model:
    """numpy / dict model of B200_expand_edges over the nine layers of each type"""

    def __init__(self, types):
        self.t = []
        for lay in types:
            h = [x.h if isinstance(x, Matrix) else x for x in (list(lay) + [None] * 9)[:9]]
            m = {(int(i), int(j)): int(v) for i, j, v in zip(*tuples(h[0], True))}
            dp = {(int(i), int(j)): int(v) for i, j, v in zip(*tuples(h[1], True))}
            dm = set(zip(*[a.astype(int).tolist() for a in tuples(h[2], False)[:2]]))
            eff = {k: v for k, v in m.items() if k not in dm}
            eff.update(dp)
            pairs = lambda x: set(zip(*[a.astype(int).tolist() for a in tuples(x, False)[:2]]))
            mt = (pairs(h[3]) - pairs(h[5])) | pairs(h[4])
            me = sorted((pairs(h[6]) - pairs(h[8])) | pairs(h[7]))
            out_rows, in_rows, ids = {}, {}, {}
            for (a, b) in sorted(eff):
                out_rows.setdefault(a, []).append(b)
            for (a, b) in sorted(mt):
                in_rows.setdefault(a, []).append(b)
            for key, eid in me:
                ids.setdefault(key, []).append(eid)
            self.t.append((eff, out_rows, in_rows, {k: set(v) for k, v in in_rows.items()}, ids))

    def ids(self, t, a, b):
        eff, ids = self.t[t][0], self.t[t][4]
        v = eff.get((a, b))
        if v is None:
            return []
        return [v] if v != MULTI else ids.get(a << 32 | b, [])

    def expand(self, src, dir, mode, targets=None):
        p, node, edge, typ, rev = [0], [], [], [], []
        blocks = {fb.DIR_OUT: (False,), fb.DIR_IN: (True,), fb.DIR_BOTH: (False, True)}[dir]
        for i, s in enumerate(int(x) for x in src):
            for r in blocks:
                cand = sorted(set().union(*[set(t[2 if r else 1].get(s, ())) for t in self.t]))
                if targets is not None:
                    cand = [x for x in cand if x == int(targets[i])]
                for x in cand:
                    if r and dir == fb.DIR_BOTH and x == s:
                        continue
                    done = False
                    for t in range(len(self.t)):
                        if r and x not in self.t[t][3].get(s, ()):
                            continue
                        for eid in (self.ids(t, x, s) if r else self.ids(t, s, x)):
                            node.append(x); edge.append(eid); typ.append(t); rev.append(1 if r else 0)
                            if mode == fb.EDGES_FIRST:
                                done = True
                                break
                        if done:
                            break
            p.append(len(edge))
        return (np.array(p, np.uint64), np.array(node, np.uint32), np.array(edge, np.uint64), np.array(typ, np.uint16),
                np.array(rev, np.uint8))


def same(a, b, what):
    for name, x, y in zip(("p", "node", "edge", "type", "rev"), a, b):
        assert np.array_equal(np.asarray(x, np.uint64), np.asarray(y, np.uint64)), f"{what}: {name} differs"


def make_graph(seed, id0, hub_edges=0):
    """edges with ids id0.., ~10 % of pairs carrying 2-4 edges, self-loops, a hub HUB with hub_edges out- and in-edges (a share
    of them multi-edges); vertices >= N - 100 stay isolated"""
    rng = np.random.default_rng(seed)
    k = 60_000
    a, b = rng.integers(0, N - 100, k), rng.integers(0, N - 100, k)
    a[:50] = b[:50]                                                  # self-loops
    if hub_edges:
        hs = rng.choice(N - 100, hub_edges, replace=False)
        a = np.concatenate([a, np.full(hub_edges, HUB), hs[: hub_edges // 2]])
        b = np.concatenate([b, hs, np.full(hub_edges // 2, HUB)])
    pairs = np.unique(np.stack([a, b], 1), axis=0)
    reps = np.where(rng.random(len(pairs)) < 0.1, rng.integers(2, 5, len(pairs)), 1)
    src, dst = np.repeat(pairs[:, 0], reps), np.repeat(pairs[:, 1], reps)
    perm = rng.permutation(len(src))
    ids = np.arange(id0, id0 + len(src), dtype=np.uint64)
    return src[perm], dst[perm], ids, rng


def dirty(seed, id0, hub_edges=0):
    """a bulk-loaded tensor, then pending writes: new pairs, new edges on single and multi-edge pairs (me_dp), deletions of single
    edges (dm) and of ids of multi-edge pairs (me_dm, down to a demotion)"""
    src, dst, ids, rng = make_graph(seed, id0, hub_edges)
    t = Tensor(N, src, dst, ids)
    nxt = int(ids[-1]) + 1
    order = np.lexsort((ids, dst, src))
    s2, d2, i2 = src[order], dst[order], ids[order]
    first = np.ones(len(s2), bool)
    first[1:] = (s2[1:] != s2[:-1]) | (d2[1:] != d2[:-1])
    cnt = np.diff(np.append(np.nonzero(first)[0], len(s2)))
    single = np.nonzero(first)[0][cnt == 1]
    multi = np.nonzero(first)[0][cnt > 1]
    single, multi = single[i2[single] != id0], multi[i2[multi] != id0]      # the first id stays
    pick_s = rng.choice(single, 400, replace=False)
    pick_m = rng.choice(multi, 300, replace=False)
    new_a, new_b = rng.integers(0, N - 100, 500), rng.integers(0, N - 100, 500)
    add_s = np.concatenate([new_a, s2[pick_s[:200]], s2[pick_m[:150]], [HUB] * 20])
    add_d = np.concatenate([new_b, d2[pick_s[:200]], d2[pick_m[:150]], rng.integers(0, N - 100, 20)])
    t.add(add_s, add_d, np.arange(nxt, nxt + len(add_s)))
    # deletions: single edges never touched above, and one or all-but-one ids of multi-edge pairs
    del_id, del_s, del_d = list(i2[pick_s[200:]]), list(s2[pick_s[200:]]), list(d2[pick_s[200:]])
    for q in pick_m[150:]:
        run = q
        while run + 1 < len(s2) and not first[run + 1]:
            run += 1
        n_ids = run - q + 1
        k = 1 if rng.random() < 0.5 else n_ids - 1
        for r in range(q, q + k):
            del_id.append(i2[r]); del_s.append(s2[r]); del_d.append(d2[r])
    t.remove(del_id, del_s, del_d)
    return t


@pytest.fixture(scope="module")
def world():
    fb.init()
    ts = [dirty(1, 0, hub_edges=24_000), dirty(2, 10_000_000), dirty(3, 20_000_000)]
    rng = np.random.default_rng(9)
    src = rng.integers(0, N - 100, 1500).astype(np.uint64)
    src[:6] = [HUB, N - 1, N - 2, 5, 5, HUB]                         # the hub, isolated vertices, duplicates
    return ts, src


def check_all(types, src, dir, mode, targets=None, what="", model=None):
    lays = [t.layers() for t in types]
    got = fb.expand_edges(src, lays, dir, mode, targets)
    want = (model or Model(lays)).expand(src, dir, mode, targets)
    same(got, want, f"device vs model {what}")
    same(via_host(types, src, dir, mode, targets, route=1), want, f"Tensor::get route vs model {what}")
    same(via_host(types, src, dir, mode, targets, route=0), want, f"host mirror's expand_edges vs model {what}")
    return got


def test_every_direction_mode_and_type_set(world):
    ts, src = world
    saw = set()
    for types in ([ts[0]], [ts[1], ts[2]], ts):
        model = Model([t.layers() for t in types])
        for dir in DIRS:
            for mode in MODES:
                for k in (1, 64, 1500):
                    got = check_all(types, src[:k], dir, mode, what=f"(T={len(types)} dir={dir} mode={mode} k={k})", model=model)
                    if k == 1500 and mode == fb.EDGES_ALL:
                        hub_row = int(got[0][1] - got[0][0])
                        saw.add(hub_row > 20_000)
    assert True in saw, "the hub row never exceeded 20,000 edges"


def test_ids_zero_self_loops_and_multi_edges_are_exercised(world):
    ts, src = world
    lays = ts[0].layers()
    every = np.arange(N - 100, dtype=np.uint64)
    p, node, edge, typ, rev = fb.expand_edges(every, [lays], fb.DIR_BOTH, fb.EDGES_ALL)
    rows = np.repeat(every, np.diff(p.astype(np.int64)))
    assert (edge == 0).any(), "edge id 0 missing"
    loops = rows == node
    assert loops.any() and not (loops & (rev == 1)).any(), "self-loops appear once, in the forward block"
    fwd = rev == 0
    key = rows[fwd] * (1 << 32) + node[fwd]
    assert len(np.unique(key)) < fwd.sum(), "no multi-edge pair in the output"
    for k, name in ((1, "dp"), (2, "dm"), (4, "mt_dp"), (5, "mt_dm"), (7, "me_dp"), (8, "me_dm")):
        nv = U64()
        check(lib().GrB_Matrix_nvals(C.byref(nv), lays[k]))
        assert nv.value, f"no pending writes in {name}"


def test_targets_form(world):
    ts, src = world
    rng = np.random.default_rng(3)
    p, node, _, _, _ = fb.expand_edges(src[:200], [t.layers() for t in ts], fb.DIR_BOTH, fb.EDGES_ALL)
    rows = np.repeat(np.arange(200), np.diff(p.astype(np.int64)))
    pick = rng.choice(len(rows), 300, replace=False)
    s = np.concatenate([src[:200][rows[pick]], src[:50], [HUB, 3]])   # existing pairs, both ways; random pairs; src == dst
    d = np.concatenate([node[pick].astype(np.uint64), rng.integers(0, N, 50).astype(np.uint64), [HUB, 3]])
    for types in ([ts[0]], ts):
        model = Model([t.layers() for t in types])
        for dir in DIRS:
            for mode in MODES:
                check_all(types, s, dir, mode, targets=d, what=f"(targets T={len(types)} dir={dir} mode={mode})", model=model)


def test_bind_edge_route_agrees(world):
    ts, src = world
    want = fb.expand_edges(src[:300], [t.layers() for t in ts], fb.DIR_OUT, fb.EDGES_FIRST)
    same(via_host(ts, src[:300], fb.DIR_OUT, fb.EDGES_FIRST, route=2), want, "traverse + get route")


def test_capacity_too_small_then_retry(world):
    ts, src = world
    lays = [t.layers() for t in ts]
    want = fb.expand_edges(src[:100], lays, fb.DIR_BOTH, fb.EDGES_ALL)
    got = fb.expand_edges(src[:100], lays, fb.DIR_BOTH, fb.EDGES_ALL, capacity=1)     # GrB_INSUFFICIENT_SPACE, then rerun
    same(got, want, "after the retry")
    from falkordb_b200.grb import TensorLayers, TENSOR_LAYERS
    ls = (TensorLayers * 3)()
    for k, lay in enumerate(lays):
        for name, h in zip(TENSOR_LAYERS, lay):
            setattr(ls[k], name, h)
    s = np.ascontiguousarray(src[:100], dtype=np.uint64)
    pp, nv = np.zeros(101, np.uint64), U64(0)
    node, edge = np.zeros(4, np.uint32), np.zeros(4, np.uint64)
    assert lib().B200_expand_edges(s.ctypes.data, None, 100, ls, 3, fb.DIR_BOTH, fb.EDGES_ALL, pp.ctypes.data, node.ctypes.data,
                                   edge.ctypes.data, None, None, 4, C.byref(nv)) == -103
    assert nv.value == len(want[2]) and np.array_equal(pp, want[0]), "*nout and out_p of a too-small call"


def test_me_modified_between_calls(world):
    """the multi-edge stores' device copies follow every change: a new id on a multi-edge pair, a removed one, a raw setElement"""
    ts, _ = world
    src, dst, ids, _ = make_graph(11, 50_000_000)
    t = Tensor(N, src, dst, ids)
    order = np.lexsort((ids, dst, src))
    s2, d2, i2 = src[order], dst[order], ids[order]
    dup = np.nonzero((s2[1:] == s2[:-1]) & (d2[1:] == d2[:-1]))[0][:3]
    probe = np.unique(s2[dup])
    check_all([t], probe, fb.DIR_OUT, fb.EDGES_ALL, what="(before)")
    t.add(s2[dup], d2[dup], [90_000_000, 90_000_001, 90_000_002])
    got = check_all([t], probe, fb.DIR_OUT, fb.EDGES_ALL, what="(after an add)")
    assert {90_000_000, 90_000_001, 90_000_002} <= set(got[2].tolist())
    t.remove([i2[dup[0]]], [s2[dup[0]]], [d2[dup[0]]])
    got = check_all([t], probe, fb.DIR_OUT, fb.EDGES_ALL, what="(after a remove)")
    assert int(i2[dup[0]]) not in set(got[2].tolist())
    me_dp = t.layers()[7]
    key = int(s2[dup[1]]) << 32 | int(d2[dup[1]])
    check(lib().GrB_Matrix_setElement_BOOL(me_dp, True, key, 91_000_000))
    got = check_all([t], probe, fb.DIR_OUT, fb.EDGES_ALL, what="(after a raw setElement on me_dp)")
    assert 91_000_000 in set(got[2].tolist())


def test_device_only_base_is_not_downloaded():
    fb.init()
    src, dst, ids, _ = make_graph(12, 0, hub_edges=5_000)
    t = Tensor(N, src, dst, ids)                                      # base built on the device: no host form
    lays = t.layers()
    q = np.arange(0, N, 29, dtype=np.uint64)
    fb.reset_stats()
    got = fb.expand_edges(q, [lays], fb.DIR_BOTH, fb.EDGES_ALL, capacity=1 << 20)   # one call: no retry
    moved = fb.get_stat("d2h_bytes")
    out_bytes = 8 * (len(q) + 1) + 15 * len(got[2]) + 64
    assert moved <= out_bytes + 4096, f"{moved} bytes came back for {out_bytes} bytes of output: the base was downloaded"
    assert 16 * len(src) > out_bytes + 4096                           # a download of the base (column + value per edge) would show
    same(got, Model([lays]).expand(q, fb.DIR_BOTH, fb.EDGES_ALL), "device-only base")


def raw(n, pairs, dtype):
    m = Matrix(n, n, dtype)
    if pairs:
        I, J = [a for a, _, _ in pairs], [b for _, b, _ in pairs]
        X = [v for _, _, v in pairs] if dtype == "u64" else None
        m.build(I, J, X)
        m.wait()
    return m


def test_raw_layer_corner_cases():
    """states a Tensor's own writes do not produce: a dp entry over a dm-deleted m entry, dm entries outside m, dp shadowing a
    live m entry, a MULTI_EDGE with every id deleted, an me_dp id already in me"""
    fb.init()
    n, big = 8, 1 << 60
    key = lambda a, b: a << 32 | b
    m = raw(n, [(0, 1, 0), (0, 2, MULTI), (0, 3, 5), (1, 0, 6), (2, 2, 7), (3, 0, MULTI), (4, 1, 9)], "u64")
    dp = raw(n, [(0, 3, 11), (0, 4, 12), (4, 1, 13), (5, 0, MULTI)], "u64")
    dm = raw(n, [(0, 3, 1), (6, 6, 1), (1, 0, 1)], bool)
    fwd = {(0, 1), (0, 2), (0, 3), (2, 2), (3, 0), (4, 1), (0, 4), (5, 0), (1, 0)}
    mt = raw(n, [(b, a, 1) for a, b in fwd], bool)
    mt_dm = raw(n, [(0, 1, 1), (7, 7, 1)], bool)
    mt_dp = raw(n, [], bool)
    me = Matrix(big, big)
    me.build([key(0, 2)] * 3 + [key(3, 0)] * 2, [20, 21, 22, 30, 31])
    me_dp = Matrix(big, big)
    me_dp.build([key(0, 2), key(0, 2), key(5, 0), key(5, 0)], [21, 25, 40, 41])
    me_dm = Matrix(big, big)
    me_dm.build([key(0, 2), key(3, 0), key(3, 0)], [20, 30, 31])
    lay = [m, dp, dm, mt, mt_dp, mt_dm, me, me_dp, me_dm]
    src = np.array([0, 1, 2, 3, 4, 5, 6, 7, 0], np.uint64)
    for dir in DIRS:
        for mode in MODES:
            for types in ([lay], [lay, lay[:3] + [mt, None, None]]):
                got = fb.expand_edges(src, types, dir, mode)
                same(got, Model(types).expand(src, dir, mode), f"raw layers dir={dir} mode={mode} T={len(types)}")
            got = fb.expand_edges(src, [lay], dir, mode, targets=src[::-1].copy())
            same(got, Model([lay]).expand(src, dir, mode, src[::-1]), f"raw layers, targets dir={dir} mode={mode}")
    p, node, edge, _, _ = fb.expand_edges([0], [lay], fb.DIR_OUT, fb.EDGES_ALL)
    assert node.tolist() == [1, 2, 2, 2, 3, 4] and edge.tolist() == [0, 21, 22, 25, 11, 12]
