"""B200_reach_batch_delta: multi-source reachability over relationship operands with pending writes, A = U_t (m_t \\ dm_t) u dp_t,
exact.  Every case is compared, entries and levels, with a scipy level loop over the effective operands built on the host."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    yield
    for k, v in (("bits_mode", -1), ("pull_mode", -1), ("hot_pack", 1), ("csr_push", 1)):
        fb.set_option(k, v)


def to_dev(n, pairs, dtype=bool):
    """an n x n matrix holding `pairs` (values 1.. for UINT64)"""
    pairs = sorted(set(pairs))
    c = orc.build_matrix(n, n, np.array([a for a, _ in pairs], np.int64), np.array([b for _, b in pairs], np.int64))
    x = np.arange(1, c.nnz + 1, dtype=np.uint64) if dtype == "u64" else None
    return Matrix.import_csr(n, n, c.p.astype(np.uint64), c.j, x, dtype)


def effective(m, dp, dm):
    """(m \\ dm) u dp as a set of pairs: dp wins where dp and dm hold the same entry"""
    return (set(m) - set(dm or ())) | set(dp or ())


def ref_reach(n, ops, src, max_hops, include):
    """the level loop over A = U_t E_t: F <- F*A AND NOT R, R <- R u F, until no row finds a new vertex"""
    pairs = set().union(*[effective(*o) for o in ops])
    A = sp.csr_matrix((np.ones(len(pairs), np.int32), ([a for a, _ in pairs], [b for _, b in pairs])), shape=(n, n))
    k = len(src)
    F = sp.csr_matrix((np.ones(k, np.int32), (np.arange(k), src)), shape=(k, n))
    R = F.toarray() > 0 if include else np.zeros((k, n), bool)
    level = 0
    while max_hops is None or level < max_hops:
        Y = ((F @ A).toarray() > 0) & ~R
        if not Y.any():
            break
        R |= Y
        F = sp.csr_matrix(Y.astype(np.int32))
        level += 1
    return R, level


def dense(R, k, n):
    R.wait()
    p, j, _ = R.export_csr()
    out = np.zeros((k, n), bool)
    rows = np.repeat(np.arange(k), np.diff(p.astype(np.int64)))
    out[rows, j.astype(np.int64)] = True
    return out


def check(n, ops, dev_ops, src, max_hops, include, what=""):
    """dev_ops: (m, dp, dm) device matrices (dp / dm may be None) for the host-side pair sets in ops"""
    R, lv = fb.reach_batch(src, [o[0] for o in dev_ops], max_hops, include, deltas=[(o[1], o[2]) for o in dev_ops])
    want, wl = ref_reach(n, ops, src, max_hops, include)
    got = dense(R, len(src), n)
    assert lv == wl, f"levels {lv} != {wl} {what}"
    assert np.array_equal(got, want), f"{int((got != want).sum())} entries differ {what}"
    return got


def random_operand(rng, A, ndel, nadd, overlap, outside, both):
    """host pair sets of one operand: m = A; dm = ndel entries of A + `outside` pairs not in A + `both` pairs also put into dp;
    dp = nadd new pairs + `overlap` entries of A + the `both` pairs"""
    n = A.nrows
    rows, cols, _ = A.tuples()
    m = list(zip(rows.tolist(), cols.tolist()))
    have = set(m)
    take = rng.choice(len(m), ndel + overlap + both, replace=False)
    fresh = lambda k: [t for t in zip(rng.integers(0, n, 4 * k + 8).tolist(), rng.integers(0, n, 4 * k + 8).tolist())
                       if t not in have][:k]
    dm = [m[i] for i in take[:ndel]] + fresh(outside)
    dp = fresh(nadd) + [m[i] for i in take[ndel:ndel + overlap]]
    shared = [m[i] for i in take[ndel + overlap:]] + fresh(both)
    return m, dp + shared, dm + shared


SCALE = 11
N = 1 << SCALE


@pytest.fixture(scope="module")
def world():
    """three RMAT operands with dirty deltas: host pair sets and prepared device matrices (operand 0 UINT64 with a BOOL dm)"""
    fb.init()
    rng = np.random.default_rng(7)
    ops, dev = [], []
    for t in range(3):
        A = orc.rmat_csr(SCALE, 8, 11 + t)
        m, dp, dm = random_operand(rng, A, ndel=300, nadd=200, overlap=20, outside=20, both=10)
        ops.append((m, dp, dm))
        dtype = "u64" if t == 0 else bool
        dev.append((to_dev(N, m, dtype).prepare(), to_dev(N, dp, dtype), to_dev(N, dm)))
    A0 = orc.rmat_csr(SCALE, 8, 11)
    live = np.nonzero(np.diff(A0.p))[0]
    iso = np.nonzero(np.diff(A0.p) == 0)[0]
    src = rng.choice(live, 1025, replace=False)
    src[0] = iso[0]                                # an isolated source
    return ops, dev, src


@pytest.mark.parametrize("pull_mode", [-1, 0, 1])
@pytest.mark.parametrize("nops", [1, 2, 3])
@pytest.mark.parametrize("nsrc", [1, 64, 100, 512, 1024])
def test_frontier_path_grid(world, nsrc, nops, pull_mode):
    """W = 1..16, 1-3 operands, every pull mode, hot-set packing on and off, bounded and unbounded, with and without sources"""
    ops, dev, src = world
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", pull_mode)
    for hot in (0, 1):
        fb.set_option("hot_pack", hot)
        for max_hops in (1, 2, 3, None):
            for include in (False, True):
                check(N, ops[:nops], dev[:nops], src[:nsrc], max_hops, include,
                      f"(nsrc={nsrc} nops={nops} pull={pull_mode} hot={hot} max={max_hops} incl={include})")


@pytest.mark.parametrize("nsrc", [64, 1025])
@pytest.mark.parametrize("nops", [1, 2, 3])
def test_materialised_fallback(world, nsrc, nops):
    """bits_mode 0 and more than 1024 sources: each dirty operand is materialised once per call; bits_mode -1 with up to 1024
    sources stays in frontier form"""
    ops, dev, src = world
    for mode in (0, -1):
        fb.set_option("bits_mode", mode)
        for max_hops in (1, 3, None):
            for include in (False, True):
                check(N, ops[:nops], dev[:nops], src[:nsrc], max_hops, include, f"(bits_mode={mode} nsrc={nsrc} nops={nops})")


def test_exact_where_delta_lmxm_over_masks():
    """s->a, s->b, a->c, b->c with a->c deleted: c stays reachable through b.  delta_lmxm drops it (its AND-NOT term removes c
    whenever any deleted edge reaches c from the row), which is why the reach has a hop of its own."""
    n, s, a, b, c = 8, 0, 1, 2, 3
    m, dm = [(s, a), (s, b), (a, c), (b, c)], [(a, c)]
    for mode in (1, 0):
        fb.set_option("bits_mode", mode)
        got = check(n, [(m, [], dm)], [(to_dev(n, m), None, to_dev(n, dm))], [s], None, False, f"(bits_mode={mode})")
        assert got[0, c]
    fb.set_option("bits_mode", 1)
    F, M, DM = Matrix(1, n, bool), to_dev(n, m), to_dev(n, dm)
    F.build([0], [s])
    R = set()
    for _ in range(3):
        F.delta_lmxm_fused(M, None, DM)
        R |= {int(v) for v in dense(F, 1, n).nonzero()[1]}
    assert c not in R and R == {a, b}


@pytest.mark.parametrize("pull_mode", [-1, 0, 1])
def test_hub_column(pull_mode):
    """a column with 20,000 in-edges (several repair segments merged with RED.OR): some of them deleted, then all of them"""
    n, hub = 1 << 15, 5
    ins = list(range(100, 20100))
    m = [(k, hub) for k in ins] + [(7, k) for k in range(100, 140)] + [(hub, 9), (9, 10)]
    src = [100, 150, 7, 20099, 3]
    M = to_dev(n, m).prepare()
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", pull_mode)
    some = sorted(set([(k, hub) for k in ins[::3]] + [(k, hub) for k in range(101, 120)]))   # 7 still reaches the hub via 12x
    for dm in (some, [(k, hub) for k in ins]):
        for max_hops in (1, 2, 4, None):
            check(n, [(m, [], dm)], [(M, None, to_dev(n, dm))], src, max_hops, False, f"(|dm|={len(dm)} max={max_hops})")


def test_edge_cases():
    """an only in-edge deleted, one entry in dp and dm, dm outside m, NULL and empty deltas, isolated sources, self-loops,
    UINT64 m and dp with a BOOL dm"""
    n = 16
    m = [(0, 1), (1, 2), (2, 3), (3, 3), (4, 5), (5, 6), (0, 7)]
    cases = [
        ([], [(1, 2)]),                          # 2 (and 3) lose their only in-edge
        ([(1, 2)], [(1, 2)]),                    # the same entry in dp and dm: dp wins
        ([(0, 9)], [(0, 9), (8, 8)]),            # dp and dm share an entry outside m; (8, 8) is not in m
        ([(9, 9), (6, 9)], [(12, 13), (3, 3)]),  # a new self-loop, dm outside m, a deleted self-loop
        ([], []),                                # empty deltas
    ]
    src = [0, 4, 3, 11, 9]                       # 11 is isolated, 3 has a self-loop
    for mode in (1, 0):
        fb.set_option("bits_mode", mode)
        for pull in (-1, 0, 1):
            fb.set_option("pull_mode", pull)
            for dp, dm in cases:
                dev = (to_dev(n, m, "u64").prepare(), to_dev(n, dp, "u64"), to_dev(n, dm))
                for max_hops in (1, 2, None):
                    for include in (False, True):
                        check(n, [(m, dp, dm)], [dev], src, max_hops, include, f"(mode={mode} pull={pull} dp={dp} dm={dm})")
            # NULL deltas, and NULL entries next to a dirty operand
            M = to_dev(n, m).prepare()
            check(n, [(m, [], [])], [(M, None, None)], src, None, False, "(NULL deltas)")
            check(n, [(m, [], []), (m, [(6, 14)], [(0, 1)])], [(M, None, None), (M, to_dev(n, [(6, 14)]), to_dev(n, [(0, 1)]))],
                  src, None, True, "(a clean and a dirty operand)")


def test_hot_set_order_across_a_dirty_level():
    """a prepared matrix: hop 1 pushes the CSR frontier into the matrix's hot-set order, and the repair and dp terms of that dirty
    level address the product through its vertex -> position table (the CSR frontier is converted to bit form for the repair)"""
    rng = np.random.default_rng(3)
    A = orc.rmat_csr(12, 8, 5)
    n = A.nrows
    m, dp, dm = random_operand(rng, A, ndel=400, nadd=100, overlap=5, outside=5, both=5)
    dev = (to_dev(n, m).prepare(), to_dev(n, dp), to_dev(n, dm))
    src = rng.choice(np.nonzero(np.diff(A.p))[0], 40, replace=False)
    fb.set_option("bits_mode", 1)
    for pull in (-1, 0):
        fb.set_option("pull_mode", pull)
        check(n, [(m, dp, dm)], [dev], src, 1, False, f"(hop 1, pull={pull})")
        assert fb.get_stat("last_path") == 7, "hop 1 did not push from the CSR frontier"
        for max_hops in (2, 3, None):
            check(n, [(m, dp, dm)], [dev], src, max_hops, False, f"(pull={pull} max={max_hops})")


def test_delta_free_case_is_reach_batch(world):
    """one operand without deltas (NULL or empty) gives B200_reach_batch's reached set and levels"""
    ops, dev, src = world
    M = dev[1][0]
    empty = Matrix(N, N, bool)
    for mode in (1, 0, -1):
        fb.set_option("bits_mode", mode)
        for k in (1, 100, 1024):
            for max_hops in (2, None):
                R0, l0 = fb.reach_batch(src[:k], M, max_hops, True)
                for deltas in (None, [(None, None)], [(empty, empty)]):
                    R1, l1 = fb.reach_batch(src[:k], [M], max_hops, True, deltas=deltas)
                    assert l1 == l0 and np.array_equal(R1.digest(), R0.digest()) and R1.nvals() == R0.nvals()


def test_host_mirror_matches_the_trail_dfs():
    """var_len_reach (CondVarLenTraverse's reach fast path in the host mirror) against the DISTINCT nodes the trail DFS reaches,
    over one and two dirty tensors, both directions, min_hops 0 / 1, max_hops 1, 2, 3 and unbounded"""
    L = C.CDLL(os.path.join(ROOT, "falkordb_b200", "libfdbhost.so"))
    L.fdbh_run_test.argtypes = [C.c_char_p]
    L.fdbh_last_message.restype = C.c_char_p
    assert L.fdbh_run_test(b"var_len_reach_matches_trails") == 0, L.fdbh_last_message().decode()
