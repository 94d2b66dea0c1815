"""B200_bfs_delta: single-source BFS over relationship operands with pending writes, A = U_t (m_t \\ dm_t) u dp_t, exact.  Levels and
minimum-id parents are compared array for array with oracle.bfs on the effective union, materialised on the host."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200._lib import lib, BfsInfo, U64
from falkordb_b200.grb import Matrix

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    yield
    fb.set_option("bfs_direction", 0)
    fb.set_option("timing", 0)


def to_dev(n, pairs, dtype=bool):
    """an n x n matrix holding `pairs` (values 1.. for UINT64)"""
    pairs = sorted(set(pairs))
    c = orc.build_matrix(n, n, np.array([a for a, _ in pairs], np.int64), np.array([b for _, b in pairs], np.int64))
    x = np.arange(1, c.nnz + 1, dtype=np.uint64) if dtype == "u64" else None
    return Matrix.import_csr(n, n, c.p.astype(np.uint64), c.j, x, dtype)


def union_csr(n, ops):
    """the effective union U_t (m_t \\ dm_t) u dp_t as an oracle CSR; dp wins where dp and dm hold the same entry"""
    pairs = set()
    for m, dp, dm in ops:
        pairs |= (set(m) - set(dm or ())) | set(dp or ())
    pairs = sorted(pairs)
    return orc.build_matrix(n, n, np.array([a for a, _ in pairs], np.int64), np.array([b for _, b in pairs], np.int64))


def run(dev_ops, src, max_level=-1, dest=-1):
    info = BfsInfo()
    lv, pr, _ = fb.bfs([o[0] for o in dev_ops], src, max_level, deltas=[(o[1], o[2]) for o in dev_ops], dest=dest, info=info)
    return lv, pr, info


def check(n, ops, dev_ops, src, max_level=-1, what=""):
    lv, pr, _ = run(dev_ops, src, max_level)
    wl, wp = orc.bfs(union_csr(n, ops), src, max_level)
    assert np.array_equal(lv, wl), f"{int((lv != wl).sum())} levels differ {what}"
    assert np.array_equal(pr, wp), f"{int((pr != wp).sum())} parents differ {what}"
    return lv, pr


def random_operand(rng, A, ndel, nadd, overlap, outside, both):
    """host pair sets of one operand: m = A; dm = ndel entries of A + `outside` pairs not in A + `both` pairs also put into dp;
    dp = nadd new pairs + `overlap` entries of A + the `both` pairs"""
    n = A.nrows
    rows, cols, _ = A.tuples()
    m = list(zip(rows.tolist(), cols.tolist()))
    have = set(m)
    take = rng.choice(len(m), ndel + overlap + both, replace=False)
    fresh = lambda k: [t for t in zip(rng.integers(0, n, 4 * k + 8).tolist(), rng.integers(0, n, 4 * k + 8).tolist())
                       if t not in have and t[0] != t[1]][:k]
    dm = [m[i] for i in take[:ndel]] + fresh(outside)
    dp = fresh(nadd) + [m[i] for i in take[ndel:ndel + overlap]]
    shared = [m[i] for i in take[ndel + overlap:]] + fresh(both)
    return m, dp + shared, dm + shared


SCALE = 12
N = 1 << SCALE


@pytest.fixture(scope="module")
def world():
    """three RMAT operands with dirty deltas (operand 0 UINT64 with a BOOL dm, the others BOOL) and four non-isolated sources"""
    fb.init()
    rng = np.random.default_rng(5)
    ops, dev = [], []
    for t in range(3):
        A = orc.rmat_csr(SCALE, 6, 21 + t)
        m, dp, dm = random_operand(rng, A, ndel=800, nadd=400, overlap=30, outside=30, both=20)
        ops.append((m, dp, dm))
        dtype = "u64" if t == 0 else bool
        dev.append((to_dev(N, m, dtype), to_dev(N, dp, dtype), to_dev(N, dm)))
    A0 = orc.rmat_csr(SCALE, 6, 21)
    src = rng.choice(np.nonzero(np.diff(A0.p))[0], 4, replace=False)
    return ops, dev, src


@pytest.mark.parametrize("max_level", [-1, 1, 3])
@pytest.mark.parametrize("direction", [0, 1, 2])
@pytest.mark.parametrize("nops", [1, 2, 3])
def test_grid(world, nops, direction, max_level):
    """every direction rule (auto, top-down only, bottom-up only) gives the oracle's levels and parents"""
    ops, dev, src = world
    fb.set_option("bfs_direction", direction)
    for s in src[:2]:
        check(N, ops[:nops], dev[:nops], int(s), max_level, f"nops={nops} dir={direction} max_level={max_level} src={s}")


SMALL = 130     # three bitmap words, the last one partial


def small_case(n, ops, src, max_level=-1):
    """ops: (m, dp, dm) pair lists; every direction rule, compared with the oracle.  Returns the (level, parent) arrays."""
    dev = [(to_dev(n, m), to_dev(n, dp) if dp else None, to_dev(n, dm) if dm else None) for m, dp, dm in ops]
    out = None
    for direction in (0, 1, 2):
        fb.set_option("bfs_direction", direction)
        got = check(n, ops, dev, src, max_level, f"direction {direction}")
        if out is not None:
            assert all(np.array_equal(a, b) for a, b in zip(got, out))
        out = got
    return out


def test_edge_deleted_in_one_type_survives_in_another():
    lv, pr = small_case(SMALL, [([(0, 1), (1, 129)], None, [(0, 1)]), ([(0, 1)], None, None)], 0)
    assert lv[1] == 1 and pr[1] == 0 and lv[129] == 2 and pr[129] == 1


def test_only_path_deleted_leaves_vertex_unreached():
    lv, pr = small_case(SMALL, [([(0, 1), (1, 2), (2, 70)], None, [(1, 2)])], 0)
    assert lv[1] == 1 and lv[2] == -1 and pr[2] == -1 and lv[70] == -1 and pr[70] == -1


def test_dp_edge_gives_smaller_parent():
    lv, pr = small_case(SMALL, [([(0, 5), (0, 3), (5, 77)], [(3, 77)], None)], 0)
    assert lv[77] == 2 and pr[77] == 3


def test_deleting_the_minimum_parent_edge_lets_the_next_win():
    lv, pr = small_case(SMALL, [([(0, 2), (0, 4), (0, 6), (2, 99), (4, 99), (6, 99)], None, [(2, 99)])], 0)
    assert lv[99] == 2 and pr[99] == 4


def test_dp_and_dm_on_one_entry_keeps_it():
    lv, pr = small_case(SMALL, [([(0, 7), (7, 8)], [(7, 8)], [(7, 8), (0, 9)])], 0)      # dm (0, 9) lies outside m
    assert lv[8] == 2 and pr[8] == 7 and lv[9] == -1


def test_source_without_out_edges():
    lv, pr = small_case(SMALL, [([(0, 1), (1, 2)], [(2, 3)], [(0, 1)])], 120)
    assert lv[120] == 0 and pr[120] == 120 and (lv >= 0).sum() == 1 and (pr >= 0).sum() == 1


def test_src_equals_dest():
    dev = [(to_dev(SMALL, [(0, 1), (1, 2)]), to_dev(SMALL, [(2, 3)]), to_dev(SMALL, [(0, 5)]))]
    lv, pr, info = run(dev, 0, dest=0)
    assert lv[0] == 0 and pr[0] == 0 and (lv >= 0).sum() == 1 and info.depth == 0


def test_dest_early_exit_matches_the_materialised_union(world):
    """the dest exit stops at the same level as B200_bfs_ex on the prepared union: same arrays, every direction rule"""
    ops, dev, src = world
    U = union_csr(N, ops)
    Ud = Matrix.import_csr(N, N, U.p.astype(np.uint64), U.j).prepare()
    s = int(src[0])
    wl, _ = orc.bfs(U, s)
    dest = int(np.nonzero(wl == 2)[0][0])
    for direction in (0, 1, 2):
        fb.set_option("bfs_direction", direction)
        lv, pr, info = run(dev, s, dest=dest)
        el, ep = np.empty(N, np.int64), np.empty(N, np.int64)
        ri = BfsInfo()
        fb.check(lib().B200_bfs_ex(Ud.h, s, -1, dest, el.ctypes.data, ep.ctypes.data, 0, C.byref(ri)))
        assert np.array_equal(lv, el) and np.array_equal(pr, ep) and info.depth == ri.depth == 2
        assert lv[dest] == 2


def kstat(name):
    ms, nl, by = C.c_double(), U64(), U64()
    assert lib().B200_kernel_stats(name.encode(), C.byref(ms), C.byref(nl), C.byref(by)) == 0
    return nl.value


def test_clean_operand_is_the_prepared_engine():
    """one operand without deltas: the arrays and the direction record of B200_Matrix_prepare + B200_bfs_ex; a second call finds
    the mirror cached on the handle and launches no transpose"""
    A = fb.rmat(SCALE, 16, 3)
    B = fb.rmat(SCALE, 16, 3).prepare()
    fb.set_option("timing", 1)
    fb.reset_stats()
    for s in (1, 17):
        lv, pr, info = run([(A, None, None)], s)
        el, ep = np.empty(N, np.int64), np.empty(N, np.int64)
        ri = BfsInfo()
        fb.check(lib().B200_bfs_ex(B.h, s, -1, -1, el.ctypes.data, ep.ctypes.data, 0, C.byref(ri)))
        assert np.array_equal(lv, el) and np.array_equal(pr, ep)
        assert (info.td_levels, info.bu_levels, info.depth, info.edges) == (ri.td_levels, ri.bu_levels, ri.depth, ri.edges)
        assert info.bu_levels > 0
    assert kstat("transpose") == 1                 # the first call built A's mirror, the second reused it
    assert kstat("bfs_delta") == 0
    fb.reset_stats()
    lv, pr, _ = run([(A, Matrix(N, N), None)], 1)  # an empty delta is no delta
    assert kstat("transpose") == 0 and kstat("bfs_delta") == 0


def test_dirty_call_reuses_base_mirrors_and_leaves_operands_untouched(world):
    ops, dev, src = world
    before = [[(x.nvals(), x.digest().tolist()) for x in o] for o in dev]
    run(dev, int(src[0]))
    fb.set_option("timing", 1)
    fb.reset_stats()
    check(N, ops, dev, int(src[1]))
    assert kstat("transpose") == 6                 # dp' and dm' per operand; the bases' mirrors are cached
    assert kstat("bfs_delta") > 0 and kstat("bfs_expand") == 0
    after = [[(x.nvals(), x.digest().tolist()) for x in o] for o in dev]
    assert before == after


# ---- the algo.BFS procedure over live tensors (csrc/host/algo_bfs.hpp): the device route against the reference's route ----
HN = 700


@pytest.fixture(scope="module")
def graph():
    """two relationship types with multi-edges, pending inserts and pending deletes, and the adjacency matrix kept in step"""
    import falkordb_b200.host_mirror as hm
    fb.init()
    rng = np.random.default_rng(11)
    nid = [0]

    def ids(k):
        nid[0] += k
        return np.arange(nid[0] - k, nid[0], dtype=np.uint64)

    types, held = [], []
    for t in range(2):
        s, d = rng.integers(0, HN, 2100), rng.integers(0, HN, 2100)
        s, d = np.concatenate([s, s[:150]]), np.concatenate([d, d[:150]])        # 150 multi-edges
        e = ids(len(s))
        T = hm.Tensor(HN, s, d, e)
        rel = {int(x): (int(a), int(b)) for x, a, b in zip(e, s, d)}
        ns, nd = rng.integers(0, HN, 300), rng.integers(0, HN, 300)
        ne = ids(300)
        T.add(ns, nd, ne)                                                          # pending inserts
        rel.update({int(x): (int(a), int(b)) for x, a, b in zip(ne, ns, nd)})
        gone = rng.choice(sorted(rel), 400, replace=False)                         # pending deletes, some of one multi-edge's ids
        T.remove(gone, [rel[int(x)][0] for x in gone], [rel[int(x)][1] for x in gone])
        for x in gone:
            del rel[int(x)]
        types.append(T)
        held.append(set(rel.values()))
    adj = hm.VersionedMatrix(HN)
    for a, b in sorted(held[0] | held[1]):
        adj.set(a, b)
    outdeg = np.bincount([a for a, _ in held[0]], minlength=HN)
    src = int(np.argmax(outdeg))                                                   # the busiest source of type 0
    return adj, types, held, src


@pytest.mark.parametrize("named", [(), (0,), (0, 1)])
@pytest.mark.parametrize("want_edges", [True, False])
@pytest.mark.parametrize("max_depth", [-1, 2])
def test_algo_bfs_matches_the_reference_route(graph, named, want_edges, max_depth):
    import falkordb_b200.host_mirror as hm
    adj, types, held, src = graph
    nt = [types[k] for k in named]
    got = hm.algo_bfs(adj, types, nt, src, max_depth, want_edges, route=hm.BFS_DEVICE)
    want = hm.algo_bfs(adj, types, nt, src, max_depth, want_edges, route=hm.BFS_BY_EXTRACT)
    assert len(want[0]) > 5
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert len(got[1]) == (len(got[0]) if want_edges else 0)
    pairs = set().union(*[held[k] for k in (named or (0, 1))])
    U = orc.build_matrix(HN, HN, np.array([a for a, _ in sorted(pairs)]), np.array([b for _, b in sorted(pairs)]))
    lv, _ = orc.bfs(U, src, max_depth)
    assert np.array_equal(got[0], np.array([v for v in np.nonzero(lv >= 0)[0] if v != src], np.uint64))


def test_algo_bfs_skips_deleted_nodes(graph):
    import falkordb_b200.host_mirror as hm
    adj, types, _, src = graph
    full = hm.algo_bfs(adj, types, [], src)
    dead = [int(full[0][0]), int(full[0][len(full[0]) // 2])]
    for want_edges in (True, False):
        got = hm.algo_bfs(adj, types, [types[1]], src, -1, want_edges, deleted=dead, route=hm.BFS_DEVICE)
        want = hm.algo_bfs(adj, types, [types[1]], src, -1, want_edges, deleted=dead, route=hm.BFS_BY_EXTRACT)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert not set(dead) & set(got[0].tolist())
    with pytest.raises(RuntimeError, match="Source node not found"):
        hm.algo_bfs(adj, types, [], src, deleted=[src])
