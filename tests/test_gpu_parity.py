"""GPU parity: every CUDA path, called through the C ABI (falkordb_b200.grb -> libb200grb.so), against the CPU
oracle on the same seeded inputs.  Bit-exact: identical row pointers and column indices (and values for u64).
Also transcribes the reference's own known-answer unit tests at this boundary
(graph/src/graph/graphblas/matrix.rs:1617-1775)."""
import numpy as np
import pytest
import scipy.sparse as sp

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix, Descriptor

pytestmark = pytest.mark.gpu


def rand_csr(rng, nrows, ncols, density, values=False):
    m = sp.random(nrows, ncols, density=density, format="csr", random_state=rng,
                  data_rvs=lambda k: rng.integers(0, 5, k))
    m.data = m.data.astype(np.int64)
    return orc.CSR.from_scipy(m, values=values)


def to_dev(c, dtype=None):
    dt = dtype or ("u64" if c.x is not None else bool)
    return Matrix.import_csr(c.nrows, c.ncols, c.p.astype(np.uint64), c.j, c.x if dt == "u64" else None, dt)


def from_dev(m):
    p, j, x = m.export_csr()
    return orc.CSR(m.nrows(), m.ncols(), p, j, x)


def assert_same(dev, want, what=""):
    got = from_dev(dev)
    assert got.nrows == want.nrows and got.ncols == want.ncols, what
    assert np.array_equal(got.p, want.p), f"{what}: row pointers differ"
    assert np.array_equal(got.j, want.j), f"{what}: column indices differ"
    if want.x is not None:
        assert got.x is not None and np.array_equal(got.x, want.x), f"{what}: values differ"


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    for k, v in (("bits_mode", -1), ("pull_mode", -1), ("small_cap", 4096), ("bitmap_budget", 2 << 30),
                 ("bits_min_flops", 1 << 22)):
        fb.set_option(k, v)
    yield


# ------------------------------------------------------------------------------------------ inputs
@pytest.mark.parametrize("scale,seed", [(8, 1), (12, 1), (14, 7)])
def test_rmat_generator_matches_oracle(scale, seed):
    assert_same(fb.rmat(scale, 16, seed), orc.rmat_csr(scale, 16, seed), "rmat")


def test_build_bool_and_u64_with_duplicates():
    rng = np.random.default_rng(3)
    n = 20000
    I = rng.integers(0, 500, n).astype(np.uint64)
    J = rng.integers(0, 700, n).astype(np.uint64)
    X = rng.integers(0, 1 << 40, n).astype(np.uint64)
    m = Matrix(500, 700, bool)
    m.build(I, J)
    assert_same(m, orc.build_matrix(500, 700, I, J), "build bool")
    u = Matrix(500, 700, "u64")
    u.build(I, J, X)
    assert_same(u, orc.build_matrix(500, 700, I, J, X), "build u64 (first duplicate wins)")
    bad = Matrix(4, 4, bool)
    with pytest.raises(fb.GrbError) as e:
        bad.build([4], [0])
    assert e.value.info == -105
    m2 = Matrix(500, 700, bool)
    m2.build(I[:10], J[:10])
    with pytest.raises(fb.GrbError) as e:
        m2.build(I[:10], J[:10])          # GrB_OUTPUT_NOT_EMPTY
    assert e.value.info == -7


# ------------------------------------------------------------------------------------------ reference KATs
def test_ref_grown_preserves_entries_at_every_growth_shape():
    """matrix.rs:1617-1655"""
    r0, c0 = 64, 48
    coords = sorted({(i, (i * 7) % c0) for i in range(r0)} | {(i, (i * 11 + 3) % c0) for i in range(r0)})
    rows, cols = [c[0] for c in coords], [c[1] for c in coords]
    vals = list(range(len(coords)))
    src = Matrix(r0, c0, "u64")
    src.build(rows, cols, vals)
    src.wait()
    for nrows, ncols in [(r0, c0), (r0 * 4, c0), (r0, c0 * 4), (r0 * 4, c0 * 4), (100_000, 100_000)]:
        g = src.grown(nrows, ncols)
        g.wait()
        assert (g.nrows(), g.ncols()) == (nrows, ncols)
        assert g.nvals() == src.nvals()
        assert set(g.iter()) == set(zip(rows, cols, vals))
    assert (src.nrows(), src.ncols()) == (r0, c0) and src.nvals() == len(coords)


def test_ref_grown_keeps_bool_layers_a_pattern():
    """matrix.rs:1660-1672"""
    src = Matrix(32, 32, bool)
    src.build([0, 5, 31], [0, 7, 31])
    src.wait()
    g = src.grown(4096, 4096)
    g.wait()
    assert g.nvals() == 3
    for i, j in [(0, 0), (5, 7), (31, 31)]:
        assert g.get(i, j) is True


def test_ref_build_bool_tolerates_duplicate_pairs():
    """matrix.rs:1686-1695"""
    m = Matrix(8, 8, bool)
    m.build([1, 3, 1, 3, 1], [2, 4, 2, 4, 2])
    m.wait()
    assert m.nvals() == 2 and m.get(1, 2) is True and m.get(3, 4) is True


def test_ref_build_bool_is_iso():
    """matrix.rs:1709-1775 (first half: the scalar build is iso and smaller than a valued build)"""
    N = 4096
    rows = np.arange(N)
    cols = (rows * 7) % N
    b = Matrix(N, N, bool)
    b.build(rows, cols)
    b.wait()
    assert b.is_iso()
    u = Matrix(N, N, "u64")
    u.build(rows, cols, np.ones(N))
    u.wait()
    assert not u.is_iso() and b.memory_usage() < u.memory_usage()


# ------------------------------------------------------------------------------------------ mxm, general path
@pytest.mark.parametrize("seed", range(5))
def test_mxm_rowwise_matches_oracle(seed):
    fb.set_option("bits_mode", 0)
    rng = np.random.default_rng(seed)
    n, k, m = rng.integers(1, 400, 3)
    A = rand_csr(rng, n, k, 0.05)
    B = rand_csr(rng, k, m, 0.05, values=bool(seed & 1))    # u64 operand: values never read
    C = Matrix(n, m, bool)
    C.mxm(to_dev(A), to_dev(B))
    want, flops = orc.mxm(A, B, return_flops=True)
    assert_same(C, want, "mxm")
    assert fb.get_stat("last_flops") == flops


def test_mxm_heavy_rows_single_and_multi_wave():
    """rows above small_cap take the global-bitmap path; a tiny scratch budget forces several waves"""
    fb.set_option("bits_mode", 0)
    fb.set_option("small_cap", 512)
    A = orc.rmat_csr(12, 16, 5)
    rng = np.random.default_rng(1)
    F = rand_csr(rng, 300, A.nrows, 0.01)
    want = orc.mxm(F, A)
    dA = to_dev(A)
    for budget in (2 << 30, 3 * ((A.ncols + 31) // 32) * 4):
        fb.set_option("bitmap_budget", budget)
        C = Matrix(300, A.ncols, bool)
        C.mxm(to_dev(F), dA)
        assert_same(C, want, f"heavy rows, budget {budget}")
    # in place (C aliases the left operand, matrix.rs:935-943)
    C = to_dev(F)
    C.lmxm(dA)
    assert_same(C, want, "lmxm in place")
    # A*A on a skewed graph: every bin at once
    S = orc.rmat_csr(9, 8, 2)
    C = Matrix(S.nrows, S.ncols, bool)
    C.mxm(to_dev(S), to_dev(S))
    assert_same(C, orc.mxm(S, S), "A*A")


DESCS = [None, Descriptor.S, Descriptor.C, Descriptor.SC, Descriptor.R, Descriptor.RS, Descriptor.RC, Descriptor.RSC]


@pytest.mark.parametrize("desc", DESCS)
def test_mxm_mask_descriptor_semantics(desc):
    fb.set_option("bits_mode", 0)
    rng = np.random.default_rng(11)
    A = rand_csr(rng, 90, 70, 0.08)
    B = rand_csr(rng, 70, 110, 0.08)
    M = rand_csr(rng, 90, 110, 0.3, values=True)          # valued mask: zeros are "false" unless structural
    Cold = rand_csr(rng, 90, 110, 0.1)
    name = desc.value if desc else ""
    comp, structural, replace = "C" in name, "S" in name, "R" in name
    T = orc.mxm(A, B)
    want = orc.mask_assign(Cold, T, M, comp, structural, replace)
    C = to_dev(Cold)
    C.mxm(to_dev(A), to_dev(B), to_dev(M, "u64"), desc)
    assert_same(C, want, f"mxm desc {name}")


def test_mxm_errors():
    a, b, c = Matrix(4, 5), Matrix(6, 4), Matrix(4, 4)
    with pytest.raises(fb.GrbError) as e:
        c.mxm(a, b)
    assert e.value.info == -6


# ------------------------------------------------------------------------------------------ mxm, frontier bit-matrix path
@pytest.mark.parametrize("nsrc,pull", [(1, 0), (64, 0), (64, 1), (100, 1), (1000, 0), (1024, 1)])
def test_mxm_chain_bit_frontier_matches_oracle(nsrc, pull):
    """CondTraverse's F*A*A*A (cond_traverse.rs:600-605) in frontier form, push and pull directions"""
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", pull)
    A = orc.rmat_csr(11, 16, 3)
    n = A.nrows
    rng = np.random.default_rng(nsrc)
    src = rng.choice(n, size=nsrc, replace=False)
    Fo = orc.build_matrix(nsrc, n, np.arange(nsrc), src)
    dA = to_dev(A)
    F = Matrix(nsrc, n, bool)
    F.build(np.arange(nsrc), src)
    want, total = Fo, 0
    for hop in range(3):
        want, fl = orc.mxm(want, A, return_flops=True)
        F.lmxm(dA)
        assert fb.get_stat("last_flops") == fl, f"hop {hop} flops"
        assert F.nvals() == want.nnz, f"hop {hop} nvals (popcount, no materialise)"
    F.wait()
    assert_same(F, want, f"3-hop chain, {nsrc} sources, pull={pull}")
    assert list(F.iter(0, 0)) == [(0, int(c)) for c in want.j[want.p[0]:want.p[1]]]


# names that no longer select anything; setting them all at once must leave every result bit-exact
RETIRED_OPTIONS = {"pull_kernel": 0, "unroll": 8, "small_split": 1, "count_kernel": 0, "l2_window": 1 << 20, "l2_reset": 1,
                   "fill_kernel": 0, "fill_cap": 64}
# every combination of the pull's switches -- hot-set order and the fused prep pass on / off, L2 hints and early exit at each of
# their settings (both template branches of k_pull_small / k_pull_seg) -- then the CTA-count override, then the retired names
PULL_OPTION_SETS = ([{"hot_pack": hp, "fused_prep": fp, "hints": h, "early_exit": ee}
                     for hp in (1, 0) for fp in (1, 0) for h in (-1, 0, 1) for ee in (1, 0, 2)]
                    + [{"pull_grid": g} for g in (1, 2, 16)] + [RETIRED_OPTIONS])


@pytest.mark.parametrize("opts", PULL_OPTION_SETS)
def test_bit_frontier_kernel_variants(opts):
    """every combination of the pull's options (hot-set packing, fused prep, L2 hints, early exit), the grid size override and
    the retired kernel-selection names, which must change nothing"""
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", 1)
    for k, v in opts.items():
        fb.set_option(k, v)
    try:
        A = orc.rmat_csr(12, 16, 11)
        rng = np.random.default_rng(5)
        for nsrc in (64, 130, 200):
            src = rng.choice(A.nrows, size=nsrc, replace=False)
            F = Matrix(nsrc, A.nrows, bool)
            F.build(np.arange(nsrc), src)
            dA = to_dev(A)
            want = orc.build_matrix(nsrc, A.nrows, np.arange(nsrc), src)
            for _ in range(3):
                F.lmxm(dA)
                want = orc.mxm(want, A)
            F.wait()
            assert_same(F, want, f"variant {opts} nsrc={nsrc}")
    finally:
        for k, v in (("hot_pack", 1), ("hints", -1), ("early_exit", 1), ("pull_grid", 0), ("fused_prep", 1)):
            fb.set_option(k, v)


def test_bit_frontier_rectangular_and_auto_mode():
    rng = np.random.default_rng(9)
    F = rand_csr(rng, 70, 900, 0.02)
    B = rand_csr(rng, 900, 1300, 0.01)
    want = orc.mxm(F, B)
    for mode, pull in ((1, 0), (1, 1), (-1, -1), (0, -1)):
        fb.set_option("bits_mode", mode)
        fb.set_option("pull_mode", pull)
        fb.set_option("bits_min_flops", 1)
        C = Matrix(70, 1300, bool)
        C.mxm(to_dev(F), to_dev(B))
        assert_same(C, want, f"rectangular bits_mode={mode} pull={pull}")


@pytest.mark.parametrize("bits", [0, 1])
def test_delta_lmxm_matches_oracle(bits):
    """matrix.rs:1317-1402: dirty snapshot = 3 mxm + RSC mask + eWiseAdd"""
    fb.set_option("bits_mode", bits)
    rng = np.random.default_rng(21)
    n = 600
    m = rand_csr(rng, n, n, 0.02)
    dp = orc.mask_assign(None, rand_csr(rng, n, n, 0.004), m, comp=True, structural=True, replace=True)
    dm = orc.ewise_mult(m, rand_csr(rng, n, n, 0.3))
    F = rand_csr(rng, 40, n, 0.01)
    empty = orc.CSR.empty(n, n)
    for (d_p, d_m) in ((dp, dm), (dp, empty), (empty, dm), (empty, empty)):
        f = to_dev(F)
        f.delta_lmxm(to_dev(m), to_dev(d_p), to_dev(d_m))
        f.wait()
        assert_same(f, orc.delta_lmxm(F, m, d_p, d_m), f"delta_lmxm dp={d_p.nnz} dm={d_m.nnz} bits={bits}")


# ------------------------------------------------------------------------------------------ delta-sync algebra
@pytest.mark.parametrize("seed", range(3))
def test_ewise_transpose_select_apply(seed):
    rng = np.random.default_rng(40 + seed)
    n, m = rng.integers(50, 700, 2)
    A = rand_csr(rng, n, m, 0.05, values=True)
    B = rand_csr(rng, n, m, 0.05, values=True)
    M = rand_csr(rng, n, m, 0.2)
    # eWiseAdd u64: SECOND (b wins), fresh C  (fold, versioned_matrix.rs:921)
    C = Matrix(n, m, "u64")
    C.element_wise_add(None, to_dev(A), to_dev(B), None)
    assert_same(C, orc.ewise_add(A, B, keep_values=True), "eWiseAdd SECOND")
    # eWiseAdd bool with complemented mask + replace (fold with tombstones, versioned_matrix.rs:914-919)
    Ab, Bb = orc.pattern(A), orc.pattern(B)
    C = Matrix(n, m, bool)
    C.element_wise_add(to_dev(M), to_dev(Ab), to_dev(Bb), Descriptor.RC)
    assert_same(C, orc.mask_assign(None, orc.ewise_add(Ab, Bb), M, comp=True, replace=True), "eWiseAdd RC")
    # in place: self u= b (matrix.rs:1399)
    C = to_dev(Ab)
    C.element_wise_add(None, None, to_dev(Bb), None)
    assert_same(C, orc.ewise_add(Ab, Bb), "eWiseAdd in place")
    # eWiseMult and the tombstone form dm<mask> = mask n m, no replace (versioned_matrix.rs:428-436)
    C = Matrix(n, m, bool)
    C.element_wise_multiply(None, to_dev(Ab), to_dev(B), None)
    assert_same(C, orc.ewise_mult(Ab, B), "eWiseMult")
    dm_old = orc.ewise_mult(Ab, rand_csr(rng, n, m, 0.1))
    dm = to_dev(dm_old)
    dm.element_wise_multiply(to_dev(M), to_dev(M), to_dev(A), None)
    assert_same(dm, orc.mask_assign(dm_old, orc.ewise_mult(M, A), M), "tombstone_masked")
    assert to_dev(Ab).intersection_nvals(to_dev(B)) == orc.ewise_mult(Ab, B).nnz
    # transpose keeps type and values; involution
    T = to_dev(A).transpose()
    assert_same(T, orc.transpose(A), "transpose u64")
    assert_same(T.transpose(), A, "transpose involution")
    assert_same(to_dev(Ab).transpose(), orc.transpose(Ab), "transpose bool")
    # masked copy / set difference via GrB_transpose(..., RCT0) (matrix.rs:824-845)
    C = to_dev(A)
    C.remove_all(to_dev(M))
    assert_same(C, orc.mask_assign(None, A, M, comp=True, replace=True), "remove_all")
    C = Matrix(n, m, "u64")
    C.select(to_dev(M), to_dev(A))
    assert_same(C, orc.mask_assign(None, A, M, comp=True, replace=True), "select")
    # set_pattern: C<M,desc> u= pattern(A) as true; A's values (incl. 0) never read (matrix.rs:898-924)
    C = to_dev(Bb)
    C.set_pattern(None, to_dev(A), None)
    assert_same(C, orc.ewise_add(Bb, Ab), "set_pattern")
    C = to_dev(Bb)
    C.set_pattern(to_dev(M), to_dev(A), Descriptor.C)
    assert_same(C, orc.mask_assign(Bb, Ab, M, comp=True, accum=True), "set_pattern masked C")


def test_skewed_rows_in_set_algebra():
    """hub rows (RMAT) through the warp-per-row union / filter kernels"""
    A = orc.rmat_csr(11, 16, 1)
    B = orc.rmat_csr(11, 16, 2)
    C = Matrix(A.nrows, A.ncols, bool)
    C.element_wise_add(None, to_dev(A), to_dev(B), None)
    assert_same(C, orc.ewise_add(A, B), "union rmat")
    C = to_dev(A)
    C.remove_all(to_dev(B))
    assert_same(C, orc.mask_assign(None, A, B, comp=True, structural=True, replace=True), "difference rmat")
    assert_same(to_dev(A).transpose(), orc.transpose(A), "transpose rmat")


def test_device_resize_dup_clear_and_host_round_trip():
    rng = np.random.default_rng(5)
    A = rand_csr(rng, 200, 300, 0.05, values=True)
    d = to_dev(A)
    g = d.grown(1000, 2000)
    g.wait()
    assert g.nvals() == A.nnz and set(g.iter()) == A.tuple_set()
    s = d.dup()
    s.resize(50, 60)
    assert set(s.iter()) == {t for t in A.tuple_set() if t[0] < 50 and t[1] < 60}
    # host element writes on top of a device-resident matrix, then a bulk op sees them
    d.set(0, 0, 77)
    rr, cc = int(A.tuples()[0][-1]), int(A.tuples()[1][-1])     # the last stored tuple, never (0,0)
    assert (rr, cc) != (0, 0)
    d.remove(rr, cc)
    want = A.tuple_set()
    want = {t for t in want if (t[0], t[1]) != (rr, cc) and (t[0], t[1]) != (0, 0)}
    want.add((0, 0, 77))
    assert set(d.iter()) == want
    t = d.transpose()
    assert set(t.iter()) == {(c, r, v) for r, c, v in want}
    d.clear()
    assert d.nvals() == 0 and list(d.iter()) == []


# ------------------------------------------------------------------------------------------ BFS / frontier steps
@pytest.mark.parametrize("scale,seed", [(10, 1), (13, 4)])
def test_bfs_levels_and_min_parents(scale, seed):
    A = orc.rmat_csr(scale, 16, seed)
    dA = to_dev(A)
    deg = np.diff(A.p)
    srcs = np.nonzero(deg > 0)[0][[0, 7, 100]]
    for s in srcs:
        lvl, par, edges = fb.bfs(dA, int(s))
        wl, wp = orc.bfs(A, int(s))
        assert np.array_equal(lvl, wl), "levels"
        assert np.array_equal(par, wp), "min-id parents"
        assert edges == int(deg[wl >= 0].sum()) or edges <= int(deg[wl >= 0].sum())
        l2, _, _ = fb.bfs(dA, int(s), max_level=2, want_parent=False)
        assert np.array_equal(l2, orc.bfs(A, int(s), 2)[0])


def test_lagraph_bfs_entry_and_vxm():
    import ctypes as C
    from falkordb_b200._lib import lib, obj, P, U64
    L = lib()
    A = orc.rmat_csr(9, 8, 3)
    dA = to_dev(A)
    g = P()
    h = P(dA.h.value)
    assert L.LAGraph_New(C.byref(g), C.byref(h), 1, None) == 0 and not h.value
    lv, pv = P(), P()
    src = int(np.nonzero(np.diff(A.p))[0][0])
    assert L.LAGr_BreadthFirstSearch_Extended(C.byref(lv), C.byref(pv), g, src, -1, -1, False, None) == 0
    wl, wp = orc.bfs(A, src)
    nv = U64()
    L.GrB_Vector_nvals(C.byref(nv), lv)
    n = nv.value
    I, X = np.empty(n, np.uint64), np.empty(n, np.int64)
    cap = U64(n)
    assert L.GrB_Vector_extractTuples_INT64(I.ctypes.data, X.ctypes.data, C.byref(cap), lv) == 0
    assert np.array_equal(I, np.nonzero(wl >= 0)[0]) and np.array_equal(X, wl[wl >= 0])
    # borrowed-graph teardown (algo_procedures.rs:407-413): detach A before LAGraph_Delete
    C.cast(g, C.POINTER(P))[0] = None
    assert L.LAGraph_Delete(C.byref(g), None) == 0
    L.GrB_Vector_free(C.byref(lv)); L.GrB_Vector_free(C.byref(pv))
    # one push step via GrB_vxm equals BFS level 1
    u, w = P(), P()
    L.GrB_Vector_new(C.byref(u), obj("GrB_BOOL"), A.nrows)
    L.GrB_Vector_new(C.byref(w), obj("GrB_BOOL"), A.ncols)
    L.GrB_Vector_setElement_BOOL(u, True, src)
    assert L.GrB_vxm(w, None, None, obj("GxB_ANY_PAIR_BOOL"), u, dA.h, None) == 0
    L.GrB_Vector_nvals(C.byref(nv), w)
    I = np.empty(nv.value, np.uint64)
    cap = U64(nv.value)
    L.GrB_Vector_extractTuples_BOOL(I.ctypes.data, None, C.byref(cap), w)
    assert np.array_equal(I, A.j[A.p[src]:A.p[src + 1]])
    L.GrB_Vector_free(C.byref(u)); L.GrB_Vector_free(C.byref(w))


def test_extract_pairs_batched_probe():
    """ExpandInto (expand_into.rs:195-249): both endpoints bound -> one lookup per row, here one call per batch"""
    rng = np.random.default_rng(8)
    A = rand_csr(rng, 500, 600, 0.03, values=True)
    d = to_dev(A)
    r, c, x = A.tuples()
    pick = rng.choice(A.nnz, 300, replace=False)
    I = np.concatenate([r[pick], rng.integers(0, 500, 300).astype(np.uint64), [499, 10 ** 9]])
    J = np.concatenate([c[pick], rng.integers(0, 600, 300).astype(np.uint64), [10 ** 9, 3]])
    found, vals = d.extract_pairs(I, J)
    have = {(int(a), int(b)): int(v) for a, b, v in zip(r, c, x)}
    for t in range(len(I)):
        key = (int(I[t]), int(J[t]))
        assert found[t] == (key in have)
        if found[t]:
            assert vals[t] == have[key] == d.get(*key)
    fb_, vb = to_dev(orc.pattern(A)).extract_pairs(I[:10], J[:10])
    assert fb_.all() and (vb == 1).all()


def test_masked_mxm_fused_triangle_pattern():
    """BASELINE config 4: C<L,struct> = L*L on a symmetrised lower-triangular RMAT (edges that close a wedge); the fused
    kernel only ever evaluates the product at the mask's positions"""
    fb.set_option("bits_mode", 0)
    A = orc.rmat_csr(11, 8, 6)
    S = orc.ewise_add(A, orc.transpose(A))
    r, c, _ = S.tuples()
    keep = r > c
    L = orc.build_matrix(S.nrows, S.ncols, r[keep], c[keep])
    want = orc.mxm(L, L, L, 1)
    dL = to_dev(L)
    C = Matrix(L.nrows, L.ncols, bool)
    C.mxm(dL, dL, dL, Descriptor.S)
    assert_same(C, want, "C<L> = L*L")
    assert fb.get_stat("last_path") == 6 and want.nnz > 0
    # no-replace form keeps C's old entries outside the mask
    rng = np.random.default_rng(1)
    Cold = rand_csr(rng, L.nrows, L.ncols, 0.001)
    C2 = to_dev(Cold)
    C2.mxm(dL, dL, dL, Descriptor.S)
    assert_same(C2, orc.mask_assign(Cold, orc.mxm(L, L), L, False, True, False), "C<L> = L*L, no replace")


def bitmap_of(csr):
    """numpy restatement of the packed row-major bitmap format"""
    wpr = (csr.ncols + 63) // 64
    bm = np.zeros((csr.nrows, wpr), np.uint64)
    rows = np.repeat(np.arange(csr.nrows), np.diff(csr.p))
    np.bitwise_or.at(bm, (rows, csr.j.astype(np.int64) >> 6), np.uint64(1) << (csr.j.astype(np.uint64) & np.uint64(63)))
    return bm


@pytest.mark.parametrize("nsrc,ncols_log", [(64, 12), (100, 12), (257, 11), (1, 10)])
def test_export_bitmap_of_frontier_chain(nsrc, ncols_log):
    """the bit-matrix result of a chain leaves as a row-major bitmap without building its CSR; CSR-form matrices too"""
    fb.set_option("bits_mode", 1)
    A = orc.rmat_csr(ncols_log, 8, 21)
    rng = np.random.default_rng(nsrc)
    src = rng.choice(A.nrows, size=nsrc, replace=False)
    F = Matrix(nsrc, A.nrows, bool)
    F.build(np.arange(nsrc), src)
    dA = to_dev(A)
    want = orc.build_matrix(nsrc, A.nrows, np.arange(nsrc), src)
    for _ in range(2):
        F.lmxm(dA)
        want = orc.mxm(want, A)
    kind, bm, nv = F.export_auto()          # 2-hop results on these graphs are far denser than 1/32
    assert kind == "bitmap" and nv == want.nnz
    assert np.array_equal(bm, bitmap_of(want))
    F.wait()                                 # materialise the CSR; same answer from the CSR-form path
    assert_same(F, want, "after bitmap export")
    G = to_dev(want)
    bm2, nv2 = G.export_bitmap()
    assert nv2 == want.nnz and np.array_equal(bm2, bitmap_of(want))


def test_export_bitmap_rectangular_and_empty():
    rng = np.random.default_rng(77)
    for (m, n, d) in ((5, 130, 0.2), (70, 64, 0.5), (3, 1000, 0.0), (1025, 70, 0.05)):
        M = rand_csr(rng, m, n, d)
        bm, nv = to_dev(M).export_bitmap()
        assert nv == M.nnz and np.array_equal(bm, bitmap_of(M))
    with pytest.raises(Exception):
        lib = fb.lib()
        h = to_dev(rand_csr(rng, 4, 100, 0.1))
        out = np.zeros(4 * 5, np.uint64)
        fb.check(lib.B200_Matrix_export_bitmap(h.h, out.ctypes.data, 5, None, 0))   # wrong words_per_row


@pytest.mark.parametrize("materialise_first", [False, True])
def test_row_iterator_walks_dense_chain_result_from_bitmap(materialise_first):
    """GxB_rowIterator over a dense frontier-chain result (bitmap snapshot inside the iterator): same ascending
    (row, col) stream as the sparse walk, incl. seek into the middle, empty rows and the exhausted state"""
    fb.set_option("bits_mode", 1)
    A = orc.rmat_csr(10, 8, 5)
    rng = np.random.default_rng(12)
    nsrc = 70
    src = rng.choice(A.nrows, size=nsrc, replace=False)
    rows = np.arange(nsrc)
    keep = rows != 3                                   # row 3 stays empty
    F = Matrix(nsrc, A.nrows, bool)
    F.build(rows[keep], src[keep])
    want = orc.build_matrix(nsrc, A.nrows, rows[keep], src[keep])
    dA = to_dev(A)
    for _ in range(2):
        F.lmxm(dA)
        want = orc.mxm(want, A)
    assert want.nnz * 32 > nsrc * A.nrows              # dense enough for the bitmap walk
    if materialise_first:
        F.wait()
    wr = np.repeat(np.arange(nsrc), np.diff(want.p))
    expect = list(zip(wr.tolist(), want.j.tolist()))
    assert list(F.iter()) == expect
    assert list(F.iter(3, 5)) == [t for t in expect if 3 <= t[0] <= 5]
    assert list(F.iter(nsrc - 1)) == [t for t in expect if t[0] >= nsrc - 1]
    assert_same(F, want, "after iterating")


# early exit at each setting x hot-set order on / off x occupancy grid or one CTA per SM (fewer 8-lane groups, so each deals
# more list entries and more long-row segments), then the retired names
@pytest.mark.parametrize("opts", [{"early_exit": ee, "hot_pack": hp, "pull_grid": g} for ee in (1, 2, 0) for hp in (1, 0) for g in (0, 1)]
                         + [RETIRED_OPTIONS])
def test_pull_bins_small_mid_long_rows(opts):
    """a graph whose transpose has empty, small (<= 8), mid and long (> 4096 entries) rows, so every bin of the
    degree-binned pull (small rows, whole mid rows, segments of long rows) is exercised; W = 1, 8 and 16 word columns"""
    rng = np.random.default_rng(2024)
    n = 20000
    src, dst = [], []
    for hub, deg in ((5, 9000), (17, 6000), (19999, 4097), (300, 4096)):       # long rows and the boundary case
        s_ = rng.choice(n, size=deg, replace=False)
        src.append(s_); dst.append(np.full(deg, hub))
    for j in range(1000, 1400):                                               # mid rows, 9..500 entries
        deg = 9 + (j * 37) % 492
        src.append(rng.choice(n, size=deg, replace=False)); dst.append(np.full(deg, j))
    m = 30000                                                                 # sprinkle: rows of 0..8 entries
    src.append(rng.integers(0, n, m)); dst.append(rng.integers(2000, n, m))
    src = np.concatenate(src); dst = np.concatenate(dst)
    A = orc.build_matrix(n, n, src, dst)
    indeg = np.bincount(A.j, minlength=n)
    assert indeg.max() > 4096 and (indeg == 0).any() and ((indeg > 0) & (indeg <= 8)).any() and ((indeg > 8) & (indeg <= 4096)).any()
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", 1)
    for k, v in opts.items():
        fb.set_option(k, v)
    try:
        dA = to_dev(A)
        for nsrc in (40, 300, 1000):
            s0 = rng.choice(n, size=nsrc, replace=False)
            F = Matrix(nsrc, n, bool)
            F.build(np.arange(nsrc), s0)
            want = orc.build_matrix(nsrc, n, np.arange(nsrc), s0)
            for _ in range(3):
                F.lmxm(dA)
                want = orc.mxm(want, A)
            assert fb.get_stat("last_path") == 3, "the pull direction was not taken"
            F.wait()
            assert_same(F, want, f"binned pull {opts} nsrc={nsrc}")
    finally:
        for k, v in (("hot_pack", 1), ("early_exit", 1), ("pull_grid", 0), ("pull_mode", -1), ("bits_mode", -1)):
            fb.set_option(k, v)


@pytest.mark.parametrize("diag_filter", [1, 0])
def test_frontier_times_diagonal_label_matrix(diag_filter):
    """F*A*L with a diagonal label matrix L (graph.rs:1191): the column-filter fast path and the ordinary hop agree with
    the oracle; a non-diagonal matrix with nnz <= n must not be mistaken for one; the cached verdict follows updates"""
    fb.set_option("bits_mode", 1)
    fb.set_option("diag_filter", diag_filter)
    try:
        A = orc.rmat_csr(11, 8, 31)
        n = A.nrows
        rng = np.random.default_rng(8)
        lab = np.sort(rng.choice(n, n // 4, replace=False))
        Ld = orc.build_matrix(n, n, lab, lab)
        perm = orc.build_matrix(n, n, np.arange(n), np.roll(np.arange(n), 1))        # nnz == n but off-diagonal
        for nsrc in (50, 300):
            src = rng.choice(n, size=nsrc, replace=False)
            F = Matrix(nsrc, n, bool)
            F.build(np.arange(nsrc), src)
            want = orc.build_matrix(nsrc, n, np.arange(nsrc), src)
            dA, dL, dP = to_dev(A), to_dev(Ld), to_dev(perm)
            F.lmxm(dA); want = orc.mxm(want, A)
            F.lmxm(dA); want = orc.mxm(want, A)
            F.lmxm(dL); want = orc.mxm(want, Ld)
            assert fb.get_stat("last_path") == (5 if diag_filter else fb.get_stat("last_path"))
            assert fb.get_stat("last_flops") == want.nnz                 # every kept entry is one multiply
            F.lmxm(dP); want = orc.mxm(want, perm)
            assert fb.get_stat("last_path") != 5
            dL.set(int(lab[0]), int((lab[0] + 1) % n))                   # no longer diagonal
            F.lmxm(dL)
            L2 = orc.build_matrix(n, n, np.append(lab, lab[0]), np.append(lab, (lab[0] + 1) % n))
            want = orc.mxm(want, L2)
            assert fb.get_stat("last_path") != 5
            F.wait()
            assert_same(F, want, f"diag_filter={diag_filter} nsrc={nsrc}")
    finally:
        fb.set_option("diag_filter", 1)


@pytest.mark.parametrize("frontier_log", [None, 9])
def test_config2_single_mxm_on_rmat(frontier_log):
    """BASELINE config 2 at test scale: one GrB_mxm over ANY_PAIR on an RMAT graph, F = A (full) and F = the rows of A
    for a random frontier of 2^k vertices (the frontier path takes it when it has <= 1024 rows)"""
    A = orc.rmat_csr(13, 16, 22)
    n = A.nrows
    dA = to_dev(A)
    if frontier_log is None:
        F, dF = A, to_dev(A)
    else:
        rng = np.random.default_rng(2)
        front = np.sort(rng.choice(n, size=1 << frontier_log, replace=False))
        rows = np.repeat(np.arange(len(front)), np.diff(A.p)[front])
        cols = np.concatenate([A.j[A.p[v]:A.p[v + 1]] for v in front])
        F = orc.build_matrix(len(front), n, rows, cols)
        dF = to_dev(F)
    want = orc.mxm(F, A)
    C_ = Matrix(F.nrows, n, bool)
    C_.mxm(dF, dA)
    C_.wait()
    assert fb.get_stat("last_flops") == int(np.diff(A.p)[F.j].sum())        # flops = sum of deg_A(k) over F's entries (SURVEY 8d)
    assert_same(C_, want, f"config 2, frontier_log={frontier_log}")


def ldbc_shaped(persons, posts, tags, seed):
    """SF-shaped synthetic social graph, all matrices n x n with label ranges (graph.rs:1191, 1211): persons [0, P),
    posts [P, P+Q), tags [P+Q, n).  KNOWS power-law among persons, one creator per post (person -> post), 1-3 tags per post
    with a Zipf-like tag popularity.  Counts used are printed by the test on failure through the assertion message."""
    rng = np.random.default_rng(seed)
    n = persons + posts + tags
    deg = np.minimum(persons - 1, (rng.pareto(1.6, persons) * 6 + 1).astype(np.int64))
    ks = np.repeat(np.arange(persons), deg)
    kd = rng.integers(0, persons, len(ks))
    keep = ks != kd
    knows = orc.build_matrix(n, n, np.concatenate([ks[keep], kd[keep]]), np.concatenate([kd[keep], ks[keep]]))   # symmetric
    creator = np.minimum(persons - 1, (rng.pareto(1.2, posts) * persons / 20).astype(np.int64))
    created = orc.build_matrix(n, n, creator, persons + np.arange(posts))
    ntag = rng.integers(1, 4, posts)
    ps = np.repeat(persons + np.arange(posts), ntag)
    tg = persons + posts + np.minimum(tags - 1, (rng.pareto(1.1, len(ps)) * tags / 50).astype(np.int64))
    hastag = orc.build_matrix(n, n, ps, tg)
    return n, knows, created, hastag


@pytest.mark.parametrize("persons,posts,tags", [(700, 9000, 300), (3000, 30000, 800)])
def test_config3_three_hop_chain_over_three_relationship_matrices(persons, posts, tags):
    """BASELINE config 3 at test scale: F = all Persons; F <- F*KNOWS*CREATED*HASTAG (friends' posts' tags).  <= 1024
    persons ride the frontier bit-matrix path, more take the row-wise SpGEMM; both must match the oracle"""
    n, knows, created, hastag = ldbc_shaped(persons, posts, tags, 5)
    F = Matrix(persons, n, bool)
    F.build(np.arange(persons), np.arange(persons))
    want = orc.build_matrix(persons, n, np.arange(persons), np.arange(persons))
    for M_ in (knows, created, hastag):
        F.lmxm(to_dev(M_))
        want = orc.mxm(want, M_)
    F.wait()
    assert want.nnz > 0 and want.j.min() >= persons + posts, "the chain must land in the tag range"
    assert_same(F, want, f"config 3: persons={persons} posts={posts} tags={tags} nnz={knows.nnz},{created.nnz},{hastag.nnz}")


def test_first_hop_copy_path_for_single_entry_rows():
    """F(i, src_i) = 1 (cond_traverse.rs:600-601): the row-wise path copies rows of A instead of sorting; empty rows,
    repeated sources, sinks and a valued operand included; one extra entry anywhere must fall back to the general path"""
    fb.set_option("bits_mode", 0)
    A = orc.rmat_csr(12, 16, 77)
    n = A.nrows
    rng = np.random.default_rng(6)
    nsrc = 500
    src = rng.integers(0, n, nsrc)                      # repeats allowed, sinks included
    rows = np.arange(nsrc)
    keep = rng.random(nsrc) < 0.8                       # some rows of F stay empty
    F = orc.build_matrix(nsrc, n, rows[keep], src[keep])
    Av = orc.CSR(n, n, A.p.copy(), A.j.copy(), np.arange(A.nnz, dtype=np.uint64) + 5)      # u64 operand: values never read
    for B in (A, Av):
        C_ = Matrix(nsrc, n, bool)
        C_.mxm(to_dev(F), to_dev(B))
        assert_same(C_, orc.mxm(F, A), "single-entry rows")
        assert fb.get_stat("last_flops") == int(np.diff(A.p)[F.j].sum())
    F2 = orc.build_matrix(nsrc, n, np.append(rows[keep], 7), np.append(src[keep], (src[7] + 1) % n))
    C_ = Matrix(nsrc, n, bool)
    C_.mxm(to_dev(F2), to_dev(A))
    assert_same(C_, orc.mxm(F2, A), "one row with two entries")


@pytest.mark.parametrize("nsrc", [3, 64, 200, 1000])
def test_push_straight_from_a_csr_frontier(nsrc):
    """a tiny CSR frontier expands from its entries (path 7) without a bit-matrix of its own; duplicates of a source,
    sinks, a structural-complement mask (delta_lmxm's RSC form) and the decline rule for large expansions"""
    A = orc.rmat_csr(12, 8, 3)
    n = A.nrows
    rng = np.random.default_rng(nsrc)
    src = rng.integers(0, n, nsrc)
    F0 = orc.build_matrix(nsrc, n, np.arange(nsrc), src)
    dA = to_dev(A)
    for csr_push in (1, 0):
        fb.set_option("bits_mode", 1)
        fb.set_option("csr_push", csr_push)
        try:
            F = to_dev(F0)
            F.lmxm(dA)
            assert fb.get_stat("last_path") == (7 if csr_push else fb.get_stat("last_path"))
            want = orc.mxm(F0, A)
            assert fb.get_stat("last_flops") == int(np.diff(A.p)[F0.j].sum())
            assert F.nvals() == want.nnz
            F.wait()
            assert_same(F, want, f"csr push={csr_push} nsrc={nsrc}")
            # masked form C<!struct(M), replace> = F0 * A (matrix.rs:1386, GrB_DESC_RSC)
            M = rand_csr(rng, nsrc, n, 0.3)
            C_ = to_dev(F0)
            C_.mxm(C_, dA, to_dev(M), Descriptor.RSC)
            assert_same(C_, orc.mxm(F0, A, M, mask_mode=2), "masked csr push")
        finally:
            fb.set_option("csr_push", 1)
    # a dense CSR frontier must decline (flops * 4 > nnz(A)) and take the bit-matrix hop instead
    Fd = rand_csr(rng, 64, n, 0.2)
    G = to_dev(Fd)
    G.lmxm(dA)
    assert fb.get_stat("last_path") != 7
    G.wait()
    assert_same(G, orc.mxm(Fd, A), "declined csr push")


@pytest.mark.parametrize("nsrc,subs", [(256, 4), (200, 3), (64, 4), (70, 1), (1000, 5)])
def test_traverse_to_host_sliced_async_hand_off(nsrc, subs):
    """falkordb_b200.traverse_to_host: row slices of the batch, each slice's bitmap copied on the second stream while the
    next slice computes; the assembled bitmap and the flops equal the one-shot chain's"""
    import torch
    A = orc.rmat_csr(12, 8, 41)
    n = A.nrows
    rng = np.random.default_rng(nsrc * 7 + subs)
    src = rng.choice(n, size=nsrc, replace=False)
    dA = to_dev(A)
    wpr = (n + 63) // 64
    out = torch.zeros(nsrc * wpr, dtype=torch.int64).pin_memory().numpy().view(np.uint64).reshape(nsrc, wpr)
    out[:] = np.uint64(0xDEADBEEF)                          # every word must be overwritten
    fl = fb.traverse_to_host(src, dA, 3, out, subs)
    want = orc.build_matrix(nsrc, n, np.arange(nsrc), src)
    wfl = 0
    for _ in range(3):
        wfl += int(np.diff(A.p)[want.j].sum())
        want = orc.mxm(want, A)
    assert fl == wfl
    assert np.array_equal(out, bitmap_of(want))
    # tickets: waiting twice is a no-op, an un-issued ticket too
    F = to_dev(want)
    t = F.export_bitmap_async(out)
    fb.wait_ticket(t)
    fb.wait_ticket(t)
    assert np.array_equal(out, bitmap_of(want))


@pytest.mark.parametrize("nsrc,hops", [(200, 3), (64, 1), (300, 2)])
def test_traverse_batch_c_entry_formats(nsrc, hops):
    """B200_traverse_batch: the coalesced traversal as one C call -- CSR hand-off, bitmap hand-off and the automatic choice
    (bitmap iff denser than one entry per 32 slots), a too-small CSR buffer, and a chain over two different matrices"""
    A = orc.rmat_csr(11, 8, 17)
    B = orc.rmat_csr(11, 4, 18)
    n = A.nrows
    rng = np.random.default_rng(nsrc + hops)
    src = rng.choice(n, size=nsrc, replace=False)
    dA, dB = to_dev(A), to_dev(B)
    ops_dev, ops_orc = [dA, dB, dA][:hops], [A, B, A][:hops]
    want = orc.build_matrix(nsrc, n, np.arange(nsrc), src)
    wfl = 0
    for M_ in ops_orc:
        wfl += int(np.diff(M_.p)[want.j].sum())
        want = orc.mxm(want, M_)
    wpr = (n + 63) // 64
    bm = np.zeros((nsrc, wpr), np.uint64)
    p_, j_ = np.zeros(nsrc + 1, np.uint64), np.zeros(want.nnz + 5, np.uint32)
    fl, nv, fmt = fb.traverse_batch(src, ops_dev, fb.OUT_CSR, out_p=p_, out_j=j_)
    assert (fl, nv, fmt) == (wfl, want.nnz, fb.OUT_CSR)
    assert np.array_equal(p_.astype(np.int64), want.p) and np.array_equal(j_[:want.nnz], want.j)
    fl, nv, fmt = fb.traverse_batch(src, ops_dev, fb.OUT_BITMAP, out_bitmap=bm)
    assert fl == wfl and fmt == fb.OUT_BITMAP and np.array_equal(bm, bitmap_of(want))
    bm[:] = 0
    p_[:] = 0
    fl, nv, fmt = fb.traverse_batch(src, ops_dev, fb.OUT_AUTO, out_bitmap=bm, out_p=p_, out_j=j_)
    assert fmt == (fb.OUT_BITMAP if want.nnz * 32 > nsrc * n else fb.OUT_CSR) and nv == want.nnz
    if fmt == fb.OUT_BITMAP:
        assert np.array_equal(bm, bitmap_of(want))
    else:
        assert np.array_equal(p_.astype(np.int64), want.p) and np.array_equal(j_[:want.nnz], want.j)
    if want.nnz > 1:
        with pytest.raises(BufferError):
            fb.traverse_batch(src, ops_dev, fb.OUT_CSR, out_p=p_, out_j=j_[: want.nnz - 1])


@pytest.mark.parametrize("nsrc,max_hops,include", [(64, None, False), (200, 2, False), (300, None, True), (5, 1, False)])
def test_multi_source_reach_matches_levelwise_oracle(nsrc, max_hops, include):
    """variable-length reachability from many sources at once: levels of C<!R,replace> = F*A and R = R u F in frontier
    form against the same loop on the oracle (and, unbounded, against scipy's connected reachability)"""
    A = orc.rmat_csr(11, 4, 19)
    n = A.nrows
    rng = np.random.default_rng(nsrc)
    src = rng.choice(n, size=nsrc, replace=False)
    R, levels = fb.multi_source_reach(src, to_dev(A), max_hops, include)
    rows = np.arange(nsrc)
    F = orc.build_matrix(nsrc, n, rows, src)
    Ro = orc.build_matrix(nsrc, n, rows, src) if include else orc.build_matrix(nsrc, n, [], [])
    lv = 0
    while max_hops is None or lv < max_hops:
        F = orc.mxm(F, A, Ro, mask_mode=2) if Ro.nnz else orc.mxm(F, A)
        if F.nnz == 0:
            break
        Ro = orc.ewise_add(Ro, F)
        lv += 1
    assert levels == lv
    R.wait()
    assert_same(R, Ro, f"reach nsrc={nsrc} max_hops={max_hops} include={include}")
    if max_hops is None and include:
        import scipy.sparse.csgraph as cg
        dist = cg.shortest_path(A.to_scipy(), method="D", unweighted=True, indices=src)
        want_rows, want_cols = np.nonzero(np.isfinite(dist))
        gr, gc, _ = from_dev(R).tuples()
        assert np.array_equal(gr, want_rows.astype(np.uint64)) and np.array_equal(gc, want_cols.astype(np.uint64))


# ------------------------------------------------------------------------------------------ rmxm / label-restricted matrix
def diag_csr(n, ids):
    ids = np.unique(np.asarray(ids, dtype=np.uint64))
    return orc.build_matrix(n, n, ids, ids)


@pytest.mark.parametrize("bits_mode", [-1, 0])
def test_rmxm_and_label_restricted_relationship_matrix(bits_mode):
    """Matrix::rmxm (matrix.rs:951-968: C = B*C, C aliases the RIGHT input) and its one caller, Graph::build_relationship_matrix
    (graph.rs:2564-2630): m = R1 (+) R2; m.rmxm(L_src1 (*) L_src2); m.lmxm(L_dst) with n x n diagonal label matrices --
    statement for statement, against the oracle composed the same way."""
    fb.set_option("bits_mode", bits_mode)
    rng = np.random.default_rng(77)
    R1 = orc.rmat_csr(12, 8, 5)
    n = R1.nrows
    R2 = rand_csr(rng, n, n, 0.001)
    ls1 = diag_csr(n, rng.choice(n, n // 2, replace=False))
    ls2 = diag_csr(n, rng.choice(n, n // 2, replace=False))
    ld = diag_csr(n, rng.choice(n, n // 3, replace=False))
    # oracle
    want = orc.ewise_add(R1, R2)
    src = orc.ewise_mult(ls1, ls2)
    want = orc.mxm(src, want)                      # rmxm: src on the left
    want = orc.mxm(want, ld)                       # lmxm: dst labels on the right
    keep_rows = set(np.nonzero(np.diff(src.p))[0].tolist())
    assert want.nnz > 0 and all((r in keep_rows) for r in np.nonzero(np.diff(want.p))[0].tolist())
    # device, through the C ABI, the reference's statements
    m = to_dev(R1)
    m.element_wise_add(None, None, to_dev(R2), None)
    s = to_dev(ls1)
    s.element_wise_multiply(None, None, to_dev(ls2), None)
    m.rmxm(s)
    assert_same(m, orc.mxm(src, orc.ewise_add(R1, R2)), "rmxm with the intersected source-label diagonal")
    m.lmxm(to_dev(ld))
    assert_same(m, want, "L_src * R * L_dst")
    # rmxm with a non-diagonal left operand, result aliasing the right input, rectangular
    B = rand_csr(rng, 300, 500, 0.02)
    Cm = rand_csr(rng, 500, 260, 0.03)
    c = to_dev(Cm)
    wantc = orc.mxm(B, Cm)
    c2 = Matrix(300, 260, bool)
    c2.mxm(to_dev(B), c)
    assert_same(c2, wantc, "B*C into a fresh output")
    sq = rand_csr(rng, 400, 400, 0.02)
    d = to_dev(sq)
    d.rmxm(to_dev(sq))                             # C = B*C with B == C's old value (A*A through the alias)
    assert_same(d, orc.mxm(sq, sq), "rmxm aliasing")
    fb.set_option("bits_mode", -1)
