"""algo.cu against exact references: FP64 mxv / vxm (PLUS_TIMES, PLUS_SECOND), LAGr_PageRank, LAGr_ConnectedComponents and
LAGraph_cdlp at sizes that reach every kernel's second grid sweep, with signed, cancelling, non-finite and subnormal values and on
degenerate graphs.

References, each checked on the CPU below before a GPU test relies on it:
  * a per-row exact sum: Dekker's TwoProduct splits every a*x into a double pair, math.fsum of the pairs is the correctly rounded
    exact sum (checked against fractions.Fraction);
  * LAGraph's PageRank recurrence in np.longdouble (checked against Fraction and against oracle.pagerank);
  * a plain-Python union-find and Counter-based CDLP for small graphs; above 2,000 vertices oracle.wcc, and a one-sort-per-round
    CDLP checked against oracle.cdlp (oracle.cdlp itself takes seconds per round at a million vertices).

Bounds (u = 2^-53, gamma_k = k u / (1 - k u)); each is derived from the kernel's arithmetic, not measured:
  * mxv row: |s^ - s| <= gamma_k * sum|a x| with k = ceil(len/8) + 6: one product rounding, ceil(len/8) lane adds, the 4-2-1 xor
    tree and `y + init + acc` (nvcc's FMA contraction of `acc += a * x` only removes roundings).
  * PageRank: max_i |r^_i - r_i| / r_i <= 8 (ceil(din/8) + ceil(n/2^18) + 32) u: the in-row sum above, the sink reduction
    (ceil(n/2^18) strided adds per thread and two 8-level trees), the divide and the teleport; 8 >= 1/(1 - 0.85) covers the
    per-iteration errors that the damped iteration carries forward.  The sequential oracle has din for ceil(din/8) and its
    sequential sink sum has the number of sinks for ceil(n/2^18).

Sweep sizes come from the device: the 8-lane kernels (k_mxv_fp64, k_cc_hook, k_cdlp_keys) cover num_sms * 1024 rows per grid sweep,
the one-thread-per-vertex kernels (k_pr_init, k_pr_scale, k_cc_jump, k_cdlp_pick) num_sms * 4096, and k_red_stage1's strided loop
runs more than once per thread above 1024 * 256 vertices.  N_BIG = 2 * num_sms * 4096 + 7 is past all three."""
import ctypes as C
import math
from collections import Counter
from fractions import Fraction

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200._lib import lib, obj, check, P

U = 2.0 ** -53
DAMPING = float(np.float32(0.85))          # LAGr_PageRank takes float damping / tol (lagraph_bindings.rs:554-555)
HAS_LONGDOUBLE = np.finfo(np.longdouble).nmant >= 63


def gamma(k):
    return k * U / (1 - k * U)


# ------------------------------------------------------------------------------------------ exact per-row sums
def _split(a):
    c = 134217729.0 * a                     # 2^27 + 1: Veltkamp split into two 26-bit halves
    hi = c - (c - a)
    return hi, a - hi


def two_product(a, b):
    """(p, e) with p + e == a * b exactly (Dekker), elementwise; finite inputs without overflow or underflow"""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    return p, e


def exact_row_sums(p, a, x):
    """correctly rounded sum over each CSR row of a[q] * x[q] (x already gathered per entry)"""
    prod, err = two_product(np.asarray(a, np.float64), np.asarray(x, np.float64))
    out = np.zeros(len(p) - 1)
    for i in np.nonzero(np.diff(p))[0]:
        s, e = p[i], p[i + 1]
        out[i] = math.fsum(prod[s:e].tolist() + err[s:e].tolist())
    return out


def row_bound(p, a, x):
    """gamma_{ceil(len/8)+6} * sum|a x| per row"""
    lens = np.diff(p)
    rows = np.repeat(np.arange(len(lens)), lens)
    sabs = np.bincount(rows, weights=np.abs(a * x), minlength=len(lens))
    return gamma(-(-lens // 8) + 6) * sabs


def test_exact_row_sums_against_fractions():
    rng = np.random.default_rng(11)
    nrows = 3000
    lens = rng.integers(1, 25, nrows)
    p = np.concatenate([[0], np.cumsum(lens)])
    m = int(p[-1])
    a = rng.standard_normal(m) * 10.0 ** rng.integers(-8, 9, m)
    x = rng.standard_normal(m) * 10.0 ** rng.integers(-8, 9, m)
    for i in range(0, nrows, 3):                  # every third row cancels catastrophically: +-1e15 pairs and small terms
        s = p[i]
        if lens[i] >= 3:
            a[s], x[s] = 1e15 * (1 + rng.random()), 1.0 + rng.random()
            a[s + 1], x[s + 1] = -a[s] * x[s] / 3.0, 3.0
    got = exact_row_sums(p, a, x)
    for i in range(nrows):
        s, e = p[i], p[i + 1]
        want = float(sum(Fraction(float(a[q])) * Fraction(float(x[q])) for q in range(s, e)))
        assert got[i] == want, (i, got[i], want)


# ------------------------------------------------------------------------------------------ PageRank in extended precision
def pagerank_ld(A, damping=DAMPING, tol=0.0, itermax=30):
    """LAGraph's recurrence in long double: d = max(outdeg, 1) / damping, the sinks' rank into the teleport, rdiff = sum|t - r|.
    Returns (r, iterations, rdiff after each iteration)."""
    ld = np.longdouble
    n = A.nrows
    if n == 0:
        return np.zeros(0, ld), 0, []
    deg = np.diff(A.p)
    src = np.repeat(np.arange(n, dtype=np.int64), deg)[np.argsort(A.j, kind="stable")]     # AT's entries, grouped by row
    atp = np.concatenate([[0], np.cumsum(np.bincount(A.j.astype(np.int64), minlength=n))])
    nonempty = atp[:-1] < atp[1:]
    dmp = ld(damping)
    d = np.maximum(deg, 1).astype(ld) / dmp
    sink = deg == 0
    r = np.full(n, ld(1) / ld(n))
    rdiffs, it, rdiff = [], 0, ld(1)
    while it < itermax and rdiff > tol:
        teleport = (ld(1) - dmp) / ld(n) + dmp / ld(n) * r[sink].sum()
        w = r / d
        acc = np.zeros(n, ld)
        if len(src):
            acc[nonempty] = np.add.reduceat(w[src], atp[:-1][nonempty])
        new = teleport + acc
        rdiff = np.abs(new - r).sum()
        r, it = new, it + 1
        rdiffs.append(rdiff)
    return r, it, rdiffs


def pagerank_fraction(n, edges, damping, iters):
    dm = Fraction(damping)
    deg = [0] * n
    for a, _ in edges:
        deg[a] += 1
    r = [Fraction(1, n)] * n
    for _ in range(iters):
        teleport = (1 - dm) / n + dm / n * sum(r[i] for i in range(n) if deg[i] == 0)
        new = [teleport] * n
        for a, b in edges:
            new[b] += r[a] * dm / deg[a]
        r = new
    return r


def pr_bound(din, n):
    return 8 * (-(-din // 8) + -(-n // (1 << 18)) + 32) * U


def max_in_degree(A):
    return int(np.bincount(A.j.astype(np.int64), minlength=max(A.nrows, 1)).max()) if A.nnz else 0


@pytest.mark.skipif(not HAS_LONGDOUBLE, reason="long double has fewer than 63 mantissa bits here")
def test_pagerank_longdouble_against_fractions_and_the_oracle():
    rng = np.random.default_rng(3)
    for n in (1, 2, 5, 9, 12):
        for trial in range(3):
            m = int(rng.integers(0, 3 * n + 1))
            pairs = sorted({(int(a), int(b)) for a, b in zip(rng.integers(0, n, m), rng.integers(0, n, m))})   # self-loops kept
            A = orc.build_matrix(n, n, [a for a, _ in pairs], [b for _, b in pairs])
            r, it, _ = pagerank_ld(A, DAMPING, 0.0, 5)
            want = pagerank_fraction(n, pairs, DAMPING, it)
            for i in range(n):
                got = Fraction(*r[i].as_integer_ratio())
                assert abs(got - want[i]) / want[i] < Fraction(1, 10 ** 17), (n, trial, i)
    for A in (orc.rmat_csr(10, 8, 3), orc.rmat_csr(8, 4, 1)):
        r, it, _ = pagerank_ld(A, DAMPING, 0.0, 30)
        want, wit = orc.pagerank(A, DAMPING, 0.0, 30)
        assert it == wit == 30
        assert np.max(np.abs(r.astype(np.float64) - want) / want) <= 1e-13
        assert abs(float(r.sum()) - 1.0) < 1e-15


# ------------------------------------------------------------------------------------------ WCC / CDLP in plain Python
def wcc_py(n, pairs):
    parent = list(range(n))

    def find(v):
        while parent[v] != v:
            parent[v] = parent[parent[v]]
            v = parent[v]
        return v
    for a, b in pairs:
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)          # the root is always the smallest id of its set
    return [find(v) for v in range(n)]


def cdlp_py(n, pairs, itermax):
    adj = [[] for _ in range(n)]
    for a, b in sorted({(a, b) for x, y in pairs for a, b in ((x, y), (y, x))}):     # the symmetric pattern, no duplicates
        adj[a].append(b)
    L, rounds = list(range(n)), 0
    if not pairs:
        return L, 0
    while rounds < itermax:
        new = list(L)
        for v in range(n):
            if adj[v]:
                c = Counter(L[u] for u in adj[v])
                top = max(c.values())
                new[v] = min(lab for lab, k in c.items() if k == top)
        rounds += 1
        same = new == L
        L = new
        if same:
            break
    return L, rounds


def uniq(key):
    """np.unique for int64 keys, by one sort (np.unique is many times slower on arrays of millions)"""
    key = np.sort(key)
    keep = np.ones(len(key), bool)
    keep[1:] = key[1:] != key[:-1]
    return key[keep]


def sym_csr(n, a, b):
    """symmetric pattern CSR of the undirected edges (a, b), duplicates merged"""
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    key = uniq(np.concatenate([a * n + b, b * n + a]))
    rows = key // n
    return orc.CSR(n, n, np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))]), (key % n).astype(np.uint32))


def test_python_wcc_and_cdlp_agree_with_the_oracle():
    rng = np.random.default_rng(8)
    for n, m in ((1, 1), (7, 4), (200, 150), (2000, 1500)):
        a, b = rng.integers(0, n, m), rng.integers(0, n, m)
        pairs = sorted({(int(x), int(y)) for x, y in zip(a, b)})
        S = sym_csr(n, a, b)
        assert np.array_equal(wcc_py(n, pairs), orc.wcc(S))
        for itermax in (0, 1, 4):
            L, rounds = cdlp_py(n, pairs, itermax)
            W, wr = orc.cdlp(S, itermax)
            assert np.array_equal(L, W) and rounds == wr, (n, itermax)
    for n in (5000, (1 << 16) + 1):
        a = np.arange(n, dtype=np.int64)
        S = sym_csr(n, np.concatenate([a, a]), rng.integers(0, n, 2 * n))
        states = cdlp_sorted(S, 6)
        for itermax in (0, 1, 6):
            W, wr = orc.cdlp(S, itermax)
            assert np.array_equal(states[min(itermax, len(states) - 1)], W) and min(itermax, len(states) - 1) == wr


def cdlp_sorted(S, itermax):
    """LAGraph_cdlp with one sort per round, vectorised (orc.cdlp's np.unique takes seconds per round at a million vertices).
    Returns the labels after 0, 1, ... rounds, stopping after itermax rounds or at the first round that changes nothing."""
    n = S.nrows
    L = np.arange(n, dtype=np.int64)
    states = [L]
    if S.nnz == 0:
        return states
    bits = max(1, (n - 1).bit_length())
    rows = np.repeat(np.arange(n, dtype=np.int64), np.diff(S.p))
    j = S.j.astype(np.int64)
    for _ in range(itermax):
        key = np.sort((rows << bits) | L[j])
        st = np.nonzero(np.concatenate([[True], key[1:] != key[:-1]]))[0]       # runs of one (row, label)
        run = np.diff(np.append(st, len(key)))
        rrow, rlab = key[st] >> bits, key[st] & ((1 << bits) - 1)
        rs = np.nonzero(np.concatenate([[True], rrow[1:] != rrow[:-1]]))[0]     # each row's first run
        top = np.repeat(np.maximum.reduceat(run, rs), np.diff(np.append(rs, len(run))))
        cand = np.nonzero(run == top)[0]                                         # longest runs; labels ascend within a row
        first = cand[np.concatenate([[True], rrow[cand][1:] != rrow[cand][:-1]])]
        new = L.copy()
        new[rrow[first]] = rlab[first]
        states.append(new)
        if np.array_equal(new, L):
            break
        L = new
    return states


# ------------------------------------------------------------------------------------------ the UINT64 -> FP64 typecast (CPU)
def test_uint64_entries_at_or_above_2_63_read_back_as_positive_doubles():
    """a sparse GrB_UINT64 entry >= 2^63 keeps its value when read as FP64 (the entries are stored in a signed 64-bit array)"""
    L = lib()
    v = P()
    check(L.GrB_Vector_new(C.byref(v), obj("GrB_UINT64"), 4))
    vals = [2 ** 63 + 2 ** 11, 2 ** 64 - 2 ** 11, 7]
    for i, x in enumerate(vals):
        check(L.GrB_Vector_setElement_UINT64(v, x, i))
    for i, x in enumerate(vals):
        got = C.c_double()
        check(L.GrB_Vector_extractElement_FP64(C.byref(got), v, i))
        assert got.value == float(x), (i, got.value)
    I, X = vec_tuples(L, v, 4)
    assert I.tolist() == [0, 1, 2] and X.tolist() == [float(x) for x in vals]
    L.GrB_Vector_free(C.byref(v))


# ------------------------------------------------------------------------------------------ C ABI helpers
def vec_tuples(L, v, n):
    nv = C.c_uint64(n)
    I, X = np.empty(max(n, 1), np.uint64), np.empty(max(n, 1), np.float64)
    check(L.GrB_Vector_extractTuples_FP64(I.ctypes.data, X.ctypes.data, C.byref(nv), v))
    return I[: nv.value].astype(np.int64), X[: nv.value]


def fp64_vec(L, n, idx, vals):
    v = P()
    check(L.GrB_Vector_new(C.byref(v), obj("GrB_FP64"), n))
    for i, x in zip(np.asarray(idx).tolist(), np.asarray(vals, np.float64).tolist()):
        check(L.GrB_Vector_setElement_FP64(v, x, i))
    return v


_libc = C.CDLL(None)
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]


def loaded_vec(L, arr, tname):
    """a full vector that adopts a copy of `arr` through GxB_Vector_load"""
    L.GxB_Vector_load.argtypes = [P, C.POINTER(P), P, C.c_uint64, C.c_uint64, C.c_int, P]
    L.GxB_Vector_load.restype = C.c_int
    arr = np.ascontiguousarray(arr)
    v = P()
    check(L.GrB_Vector_new(C.byref(v), obj(tname), len(arr)))
    buf = P(_libc.malloc(max(arr.nbytes, 1)))
    C.memmove(buf, arr.ctypes.data, arr.nbytes)
    check(L.GxB_Vector_load(v, C.byref(buf), obj(tname), len(arr), arr.nbytes, 0, None))
    return v


def fp64_mat(L, nrows, ncols, rows, cols, vals):
    m = P()
    check(L.GrB_Matrix_new(C.byref(m), obj("GrB_FP64"), nrows, ncols))
    I = np.ascontiguousarray(rows, np.uint64)
    J = np.ascontiguousarray(cols, np.uint64)
    X = np.ascontiguousarray(vals, np.float64)
    check(L.GrB_Matrix_build_FP64(m, I.ctypes.data, J.ctypes.data, X.ctypes.data, len(X), None))
    return m


def free_all(L, vecs=(), mats=()):
    for v in vecs:
        L.GrB_Vector_free(C.byref(v))
    for m in mats:
        L.GrB_Matrix_free(C.byref(m))


OPS = {   # name -> (GrB_mxv?, descriptor, streams A' instead of A)
    "mxv": (True, None, False), "mxv_T0": (True, "GrB_DESC_T0", True),
    "vxm": (False, None, True), "vxm_T1": (False, "GrB_DESC_T1", False),
}
SEMIRINGS = {"plus_times": "GrB_PLUS_TIMES_SEMIRING_FP64", "plus_second": "GxB_PLUS_SECOND_FP64"}


def run_op(L, op, sr, w, dA, u, accum=False):
    is_mxv, desc, _ = OPS[op]
    acc = obj("GrB_PLUS_FP64") if accum else None
    d = obj(desc) if desc else None
    if is_mxv:
        check(L.GrB_mxv(w, None, acc, obj(SEMIRINGS[sr]), dA, u, d))
    else:
        check(L.GrB_vxm(w, None, acc, obj(SEMIRINGS[sr]), u, dA, d))


@pytest.fixture(scope="module")
def dev():
    fb.init()
    L = lib()
    assert L.B200_stream()                          # device bring-up: num_sms is read from the device
    sms = int(fb.get_stat("num_sms"))
    return L, sms, 2 * sms * 4096 + 7


# ------------------------------------------------------------------------------------------ FP64 mxv / vxm
@pytest.mark.gpu
def test_mxv_vxm_integer_valued_exact_at_n_big(dev):
    """integer-valued operands: every partial sum is an integer below 2^53, so each result must equal the int64 reference bit for
    bit -- on every row of every grid sweep, through all four operand orientations, both semirings, dense and 30 % present u,
    and PLUS accumulation into a w that has entries where the product is absent"""
    import scipy.sparse as sp
    L, _, nb = dev
    rng = np.random.default_rng(2024)
    nrows, ncols = nb, nb + 4099                  # rectangular: the transposed cases stream ncols rows
    deg = rng.poisson(8, nrows)
    deg[rng.random(nrows) < 0.03] = 0             # empty rows: products absent even for a dense u
    long_rows = rng.choice(nrows, 3, replace=False)
    deg[long_rows] = (10_000, 50_000, 200_000)
    rows = np.repeat(np.arange(nrows, dtype=np.int64), deg)
    allowed = np.nonzero(rng.random(ncols) >= 0.03)[0]          # 3 % of the columns stay empty
    cols = allowed[rng.integers(0, len(allowed), len(rows))]
    hubs = allowed[rng.choice(len(allowed), 3, replace=False)]  # long columns for the transposed cases
    for h, k in zip(hubs, (10_000, 60_000, 200_000)):
        rows = np.concatenate([rows, rng.choice(nrows, k, replace=False)])
        cols = np.concatenate([cols, np.full(k, h)])
    key = uniq(rows * ncols + cols)
    rows, cols = key // ncols, key % ncols
    del key
    vals = rng.integers(-1024, 1025, len(rows))
    dA = fp64_mat(L, nrows, ncols, rows, cols, vals.astype(np.float64))
    M = sp.csr_matrix((vals, (rows, cols)), shape=(nrows, ncols))
    Pm = sp.csr_matrix((np.ones(len(rows), np.int64), (rows, cols)), shape=(nrows, ncols))
    del rows, cols, vals
    for op, (_, _, tr) in OPS.items():
        inner, outer = (nrows, ncols) if tr else (ncols, nrows)
        x = rng.integers(-1024, 1025, inner)
        pres = rng.random(inner) < 0.3
        Ms, Ps = (M.T.tocsr(), Pm.T.tocsr()) if tr else (M, Pm)
        u_dense = loaded_vec(L, x.astype(np.int64), "GrB_INT64")
        u_sparse = fp64_vec(L, inner, np.nonzero(pres)[0], x[pres])
        widx = np.unique(np.concatenate([rng.choice(outer, outer // 100, replace=False),
                                         np.nonzero(np.diff(Ps.indptr) == 0)[0][:2000]]))
        wval = rng.integers(-1024, 1025, len(widx))
        for sr in SEMIRINGS:
            for u, present in ((u_dense, np.ones(inner, bool)), (u_sparse, pres)):
                xp = np.where(present, x, 0)
                want = (Ms if sr == "plus_times" else Ps) @ xp
                wpres = (Ps @ present.astype(np.int64)) > 0
                for accum in (False, True):
                    w = fp64_vec(L, outer, widx, wval) if accum else fp64_vec(L, outer, [], [])
                    run_op(L, op, sr, w, dA, u, accum)
                    I, X = vec_tuples(L, w, outer)
                    ref, keep = want.copy(), wpres.copy()
                    if accum:
                        ref[widx] += wval
                        keep[widx] = True
                    tag = f"{op} {sr} {'dense' if present.all() else 'sparse'} u accum={accum}"
                    assert np.array_equal(I, np.nonzero(keep)[0]), f"{tag}: pattern"
                    assert np.array_equal(X, ref[keep].astype(np.float64)), f"{tag}: values"
                    free_all(L, [w])
        free_all(L, [u_dense, u_sparse])
    free_all(L, mats=[dA])


GRID_LENS = [0, 1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 257, 1000, 4097]


def _grid_matrix(rng, ncols, present):
    """rows of the listed lengths (about 100 of each, interleaved so that the four 8-lane groups of a warp differ), one row of
    2e5 entries and rows of +-1e15 pairs that cancel to small terms"""
    order = [GRID_LENS[(7 * i) % len(GRID_LENS)] for i in range(len(GRID_LENS))]
    lens = np.array(order * 100 + [200_000], np.int64)
    rows = np.repeat(np.arange(len(lens)), lens)
    pos = np.arange(len(rows)) - np.repeat(np.cumsum(lens) - lens, lens)
    start = rng.integers(0, ncols, len(lens))
    stride = np.maximum(1, (ncols - 1) // np.maximum(lens - 1, 1))
    stride = rng.integers(1, stride + 1)
    cols = (np.repeat(start, lens) + pos * np.repeat(stride, lens)) % ncols
    vals = rng.standard_normal(len(rows))
    # cancelling rows: pairs a, -a' with a x ~ +-1e15, over present columns, then N(0,1) terms
    pidx = np.nonzero(present)[0]
    crows, ccols, cvals = [], [], []
    r0 = len(lens)
    for k, ln in enumerate([16, 33, 64, 257, 1000] * 8):
        c = np.sort(rng.choice(pidx, ln, replace=False))
        v = rng.standard_normal(ln)
        crows.append(np.full(ln, r0 + k))
        ccols.append(c)
        cvals.append(v)
    return rows, cols, vals, r0, crows, ccols, cvals


@pytest.mark.gpu
def test_mxv_row_length_grid_within_the_derived_bound(dev):
    L, _, _ = dev
    rng = np.random.default_rng(77)
    ncols = 262_147
    present = rng.random(ncols) < 0.7
    x = rng.standard_normal(ncols)
    rows, cols, vals, r0, crows, ccols, cvals = _grid_matrix(rng, ncols, present)
    for c, v in zip(ccols, cvals):
        half = len(c) // 2 // 2 * 2                        # pairs a x ~ +c_j, a' x' ~ -c_j, then N(0,1) terms
        cj = 1e15 * (1 + rng.random(half // 2))
        v[0:half:2] = cj / x[c[0:half:2]]
        v[1:half:2] = -cj / x[c[1:half:2]]
    rows = np.concatenate([rows] + crows)
    cols = np.concatenate([cols] + ccols)
    vals = np.concatenate([vals] + cvals)
    nrows = r0 + len(crows)
    key = rows * ncols + cols
    o = np.argsort(key, kind="stable")
    rows, cols, vals = rows[o], cols[o], vals[o]
    assert len(uniq(key)) == len(key)
    p = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=nrows))])
    dA = fp64_mat(L, nrows, ncols, rows, cols, vals)
    u = fp64_vec(L, ncols, np.nonzero(present)[0], x[present])
    w = fp64_vec(L, nrows, [], [])
    xg = np.where(present[cols], x[cols], 0.0)
    exact = exact_row_sums(p, vals, xg)
    bound = row_bound(p, vals, xg)
    has = np.bincount(rows, weights=present[cols], minlength=nrows) > 0
    for sr in ("plus_times", "plus_second"):
        a = vals if sr == "plus_times" else np.ones_like(vals)
        if sr == "plus_second":
            exact, bound = exact_row_sums(p, a, xg), row_bound(p, a, xg)
        run_op(L, "mxv", sr, w, dA, u)
        I, X = vec_tuples(L, w, nrows)
        assert np.array_equal(I, np.nonzero(has)[0]), f"{sr}: the rows with a present u entry"
        err = np.abs(X - exact[has])
        bad = np.nonzero(err > bound[has])[0]
        assert len(bad) == 0, f"{sr}: rows {I[bad][:5]} err {err[bad][:5]} bound {bound[has][bad][:5]}"
        if sr == "plus_times":
            assert np.all(np.abs(exact[r0:]) < 1e3), "the cancelling rows cancel"
    # the valued transpose: mxv(G, T0) streams the same CSR as the matrix GrB_transpose gives back
    G, G2 = P(), P()
    check(L.GrB_Matrix_new(C.byref(G), obj("GrB_FP64"), ncols, nrows))
    check(L.GrB_transpose(G, None, None, dA, None))
    check(L.GrB_Matrix_new(C.byref(G2), obj("GrB_FP64"), nrows, ncols))
    check(L.GrB_transpose(G2, None, None, G, None))
    outs = []
    for m, op in ((G, "mxv_T0"), (G2, "mxv"), (dA, "mxv")):
        run_op(L, op, "plus_times", w, m, u)
        outs.append(vec_tuples(L, w, nrows))
    for I, X in outs[1:]:
        assert np.array_equal(I, outs[0][0]) and np.array_equal(X.view(np.uint64), outs[0][1].view(np.uint64))
    free_all(L, [u, w], [dA, G, G2])


@pytest.mark.gpu
def test_mxv_special_values(dev):
    """IEEE classes: +inf, inf - inf, inf * 0, NaN in a present x, NaN and inf behind an absent x, subnormal products"""
    L, _, _ = dev
    inf, nan = float("inf"), float("nan")
    x = [1.0, 2.0, 0.0, nan, nan, 1e-10, 3.0, -5.0, 1e-10]
    absent = [4, 7]
    entries = [(0, 0, inf), (0, 1, 1.0),                  # +inf
               (1, 0, inf), (1, 1, -inf),                 # inf - inf = NaN
               (2, 2, inf),                               # inf * 0 = NaN
               (3, 3, 1.0), (3, 6, 1.0),                  # NaN in a present x
               (4, 4, 5.0), (4, 6, 1.0), (4, 7, inf),     # NaN / inf behind absent x: 3.0
               (5, 5, 1e-300), (5, 8, -3e-300),           # subnormal products
               (6, 6, -inf)]                              # a single -inf term
    nrows, ncols = 8, len(x)
    r, c, v = zip(*entries)
    dA = fp64_mat(L, nrows, ncols, r, c, v)
    u = fp64_vec(L, ncols, range(ncols), x)
    for i in absent:
        check(L.GrB_Vector_removeElement(u, i))
    w = fp64_vec(L, nrows, [], [])
    run_op(L, "mxv", "plus_times", w, dA, u)
    I, X = vec_tuples(L, w, nrows)
    assert I.tolist() == [0, 1, 2, 3, 4, 5, 6], "row 7 is empty"
    assert X[0] == inf and X[6] == -inf
    assert np.isnan(X[1]) and np.isnan(X[2]) and np.isnan(X[3])
    assert X[4] == 3.0, "an absent x contributes nothing, whatever it held and whatever it meets"
    sub = 1e-300 * 1e-10 + -3e-300 * 1e-10
    assert X[5] == sub and 0 < abs(sub) < np.finfo(np.float64).tiny
    free_all(L, [u, w], [dA])


@pytest.mark.gpu
def test_mxv_operand_forms_typecasts_and_degenerate_shapes(dev):
    L, _, _ = dev
    rng = np.random.default_rng(5)
    n = 300
    m = 2400
    key = uniq(rng.integers(0, n, m) * n + rng.integers(0, n, m))
    rows, cols = key // n, key % n
    vals = rng.integers(-64, 65, len(rows)).astype(np.float64)
    dA = fp64_mat(L, n, n, rows, cols, vals)
    p = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))])
    nonempty = np.diff(p) > 0

    def check_dense(u, x, tag):
        w = fp64_vec(L, n, [], [])
        run_op(L, "mxv", "plus_times", w, dA, u)
        I, X = vec_tuples(L, w, n)
        assert np.array_equal(I, np.nonzero(nonempty)[0]), tag
        assert np.array_equal(X, exact_row_sums(p, vals, np.asarray(x, np.float64)[cols])[nonempty]), tag
        free_all(L, [w])

    xi = rng.integers(-2 ** 20, 2 ** 20, n)
    u = loaded_vec(L, xi.astype(np.int64), "GrB_INT64")
    check_dense(u, xi, "full INT64 u with negative values")
    free_all(L, [u])
    xu = rng.integers(0, 2 ** 32, n).astype(np.uint32)
    xu[:3] = (2 ** 32 - 1, 2 ** 31, 0)
    u = loaded_vec(L, xu, "GrB_UINT32")
    check_dense(u, xu.astype(np.float64), "full UINT32 u")
    free_all(L, [u])

    # sparse UINT64 at and above 2^63
    big = [2 ** 63 + 2 ** 11, 2 ** 64 - 2 ** 11]
    u = P()
    check(L.GrB_Vector_new(C.byref(u), obj("GrB_UINT64"), 2))
    for i, b in enumerate(big):
        check(L.GrB_Vector_setElement_UINT64(u, b, i))
    B = fp64_mat(L, 4, 2, [0, 1, 2, 2], [0, 1, 0, 1], [1.0, -1.0, 1.0, -1.0])
    w = fp64_vec(L, 4, [], [])
    run_op(L, "mxv", "plus_times", w, B, u)
    I, X = vec_tuples(L, w, 4)
    assert I.tolist() == [0, 1, 2] and X.tolist() == [float(big[0]), -float(big[1]), float(big[0] - big[1])]
    free_all(L, [u, w], [B])

    # BOOL u: a stored false is present with value 0.0
    u = P()
    check(L.GrB_Vector_new(C.byref(u), obj("GrB_BOOL"), 3))
    check(L.GrB_Vector_setElement_BOOL(u, False, 0))
    check(L.GrB_Vector_setElement_BOOL(u, True, 1))
    B = fp64_mat(L, 3, 3, [0, 1, 1, 2], [0, 0, 1, 2], [2.0, 2.0, 3.0, 4.0])
    w = fp64_vec(L, 3, [], [])
    for sr in SEMIRINGS:
        run_op(L, "mxv", sr, w, B, u)
        I, X = vec_tuples(L, w, 3)
        assert I.tolist() == [0, 1] and X.tolist() == ([0.0, 3.0] if sr == "plus_times" else [0.0, 1.0]), sr
    free_all(L, [u, w], [B])

    # u aliased to w, without and with accum
    x = rng.integers(-64, 65, n).astype(np.float64)
    sp_idx = np.nonzero(rng.random(n) < 0.5)[0]
    xs = np.zeros(n)
    xs[sp_idx] = x[sp_idx]
    ps = np.zeros(n, bool)
    ps[sp_idx] = True
    want = exact_row_sums(p, vals, xs[cols])
    wpres = np.bincount(rows, weights=ps[cols], minlength=n) > 0
    for accum in (False, True):
        u = fp64_vec(L, n, sp_idx, x[sp_idx])
        run_op(L, "mxv", "plus_times", u, dA, u, accum)
        I, X = vec_tuples(L, u, n)
        keep = wpres | ps if accum else wpres
        ref = want + xs if accum else want
        assert np.array_equal(I, np.nonzero(keep)[0]) and np.array_equal(X, ref[keep]), f"aliased accum={accum}"
        free_all(L, [u])

    # u = the full FP64 vector LAGr_PageRank returns
    S = orc.rmat_csr(8, 4, 2)
    assert S.nrows == 256 <= n
    u = pagerank_vector(L, S)
    _, r = vec_tuples(L, u, 256)
    B = fp64_mat(L, n, 256, rows[cols < 256], cols[cols < 256], vals[cols < 256])
    pb = np.concatenate([[0], np.cumsum(np.bincount(rows[cols < 256], minlength=n))])
    w = fp64_vec(L, n, [], [])
    run_op(L, "mxv", "plus_times", w, B, u)
    I, X = vec_tuples(L, w, n)
    xg = r[cols[cols < 256]]
    ex, bd = exact_row_sums(pb, vals[cols < 256], xg), row_bound(pb, vals[cols < 256], xg)
    assert np.array_equal(I, np.nonzero(np.diff(pb))[0]) and np.all(np.abs(X - ex[I]) <= bd[I])
    free_all(L, [u, w], [B])

    # degenerate shapes
    for nr, nc in ((0, 5), (5, 0), (1, 1), (7, 1)):
        rr = np.repeat(np.arange(nr), nc)
        cc = np.tile(np.arange(nc), nr)
        vv = np.arange(1, len(rr) + 1, dtype=np.float64) * 0.5
        Bm = fp64_mat(L, nr, nc, rr, cc, vv)
        D = np.zeros((nr, nc))
        D[rr, cc] = vv
        for op, (_, _, tr) in OPS.items():
            inner, outer = (nr, nc) if tr else (nc, nr)
            Dm = D.T if tr else D
            xv = np.arange(1, inner + 1, dtype=np.float64) * 3.0
            for accum in (False, True):
                uu = fp64_vec(L, inner, range(inner), xv)
                ww = fp64_vec(L, outer, range(outer), np.full(outer, 0.25)) if accum else fp64_vec(L, outer, [], [])
                run_op(L, op, "plus_times", ww, Bm, uu, accum)
                I, X = vec_tuples(L, ww, outer)
                has = (Dm != 0).any(axis=1) if inner else np.zeros(outer, bool)
                keep = has | accum
                ref = Dm @ xv + (0.25 if accum else 0.0)
                assert np.array_equal(I, np.nonzero(keep)[0]) and np.array_equal(X, ref[keep]), (nr, nc, op, accum)
                free_all(L, [uu, ww])
        free_all(L, mats=[Bm])
    free_all(L, mats=[dA])


# ------------------------------------------------------------------------------------------ LAGr_PageRank
def _graph(L, S, kind):
    from falkordb_b200.grb import Matrix
    m = Matrix.import_csr(S.nrows, S.ncols, S.p.astype(np.uint64), S.j, None, bool)
    G, h = P(), P(m.h.value)
    m.h = P()                                         # the matrix moves into the graph
    assert L.LAGraph_New(C.byref(G), C.byref(h), kind, None) == 0
    return G


def pagerank_vector(L, A, damping=DAMPING, tol=0.0, itermax=10):
    G = _graph(L, A, 1)
    assert L.LAGraph_Cached_AT(G, None) == 0 and L.LAGraph_Cached_OutDegree(G, None) == 0
    cen, it = P(), C.c_int(0)
    assert L.LAGr_PageRank(C.byref(cen), C.byref(it), G, damping, tol, itermax, None) == 0
    L.LAGraph_Delete(C.byref(G), None)
    return cen


def pagerank_dev(L, A, damping=DAMPING, tol=0.0, itermax=30):
    G = _graph(L, A, 1)
    assert L.LAGraph_Cached_AT(G, None) == 0 and L.LAGraph_Cached_OutDegree(G, None) == 0
    cen, it = P(), C.c_int(0)
    assert L.LAGr_PageRank(C.byref(cen), C.byref(it), G, damping, tol, itermax, None) == 0
    I, X = vec_tuples(L, cen, A.nrows)
    assert np.array_equal(I, np.arange(A.nrows)), "the centrality vector is full"
    L.GrB_Vector_free(C.byref(cen))
    L.LAGraph_Delete(C.byref(G), None)
    return X, it.value


def _csr(n, a, b):
    a = np.asarray(a, np.int64)
    b = np.asarray(b, np.int64)
    key = uniq(a * n + b)
    return orc.CSR(n, n, np.concatenate([[0], np.cumsum(np.bincount(key // n, minlength=n))]).astype(np.int64),
                   (key % n).astype(np.uint32))


def _pr_graphs():
    hub = 50_000
    R = orc.rmat_csr(10, 8, 3)
    rr, cc, _ = R.tuples()
    loops = np.arange(0, R.nrows, 3)
    return {
        "rmat10": R,
        "rmat12": orc.rmat_csr(12, 8, 5),
        "in_star": _csr(hub + 1, np.arange(1, hub + 1), np.zeros(hub, np.int64)),
        "one_non_sink": _csr(1000, np.zeros(999, np.int64), np.arange(1, 1000)),
        "self_loops": _csr(R.nrows, np.concatenate([rr, loops]), np.concatenate([cc, loops])),
        "n1": _csr(1, [], []),
        "n1_loop": _csr(1, [0], [0]),
        "n2": _csr(2, [0], [1]),
    }


@pytest.mark.gpu
@pytest.mark.skipif(not HAS_LONGDOUBLE, reason="long double has fewer than 63 mantissa bits here")
def test_pagerank_small_graphs_against_longdouble(dev):
    L, _, _ = dev
    for name, A in _pr_graphs().items():
        got, it = pagerank_dev(L, A, DAMPING, 0.0, 30)
        assert 1 <= it <= 30, f"{name}: {it} iterations"      # tol = 0 stops early only at an exact fixed point
        ref, rit, rd = pagerank_ld(A, DAMPING, 0.0, it)
        assert rit == it or rd[-1] == 0, f"{name}: the reference stops early only at an exact fixed point"
        b = pr_bound(max_in_degree(A), A.nrows)
        rel = float(np.max(np.abs(got - ref) / ref))
        assert rel <= b, f"{name}: rel err {rel} > {b}"
        assert abs(math.fsum(got.tolist()) - 1.0) <= b, f"{name}: sum {math.fsum(got.tolist())}"


@pytest.mark.gpu
@pytest.mark.skipif(not HAS_LONGDOUBLE, reason="long double has fewer than 63 mantissa bits here")
def test_pagerank_stopping_rule_matches_the_reference(dev):
    L, _, _ = dev
    for A in (orc.rmat_csr(12, 8, 5), _pr_graphs()["in_star"]):
        for tol in (1e-4, 1e-9):
            tf = float(np.float32(tol))
            _, rit, rd = pagerank_ld(A, DAMPING, tf, 1000)
            assert rit < 1000
            for k in rd[-2:]:
                assert abs(float(k) - tf) > 1e-6 * tf, "the stop is not decided by rounding"
            _, it = pagerank_dev(L, A, DAMPING, tol, 1000)
            assert it == rit, (tol, it, rit)


@pytest.mark.gpu
def test_pagerank_degenerate_inputs(dev):
    L, _, _ = dev
    got, it = pagerank_dev(L, _csr(0, [], []), DAMPING, 1e-4, 100)
    assert it == 0 and len(got) == 0
    n = 1000
    E = _csr(n, [], [])
    got, it = pagerank_dev(L, E, DAMPING, 1e-4, 30)
    _, rit, _ = pagerank_ld(E, DAMPING, float(np.float32(1e-4)), 30)
    assert it == rit and np.all(np.abs(got - 1.0 / n) <= pr_bound(0, n) / n)
    A = orc.rmat_csr(10, 8, 3)
    got, it = pagerank_dev(L, A, DAMPING, 0.0, 0)
    assert it == 0 and np.all(got == 1.0 / A.nrows)
    got, it = pagerank_dev(L, A, DAMPING, 0.0, 1)
    ref, _, _ = pagerank_ld(A, DAMPING, 0.0, 1)
    assert it == 1 and np.max(np.abs(got - ref) / ref) <= pr_bound(max_in_degree(A), A.nrows)


@pytest.mark.gpu
def test_pagerank_at_n_big(dev):
    """random graph, ~8 out-edges per vertex, 5 % sinks, one in-hub, 12 iterations: every one-thread kernel sweeps the grid
    twice and the reductions' strided loop runs 5 times per thread"""
    L, _, nb = dev
    rng = np.random.default_rng(31)
    deg = rng.poisson(8, nb)
    deg[rng.random(nb) < 0.05] = 0
    src = np.repeat(np.arange(nb, dtype=np.int64), deg)
    dst = rng.integers(0, nb, len(src))
    hub = nb // 3
    fans = rng.choice(nb, 100_000, replace=False)
    fans = fans[deg[fans] > 0]
    A = _csr(nb, np.concatenate([src, fans]), np.concatenate([dst, np.full(len(fans), hub)]))
    del src, dst
    got, it = pagerank_dev(L, A, DAMPING, 0.0, 12)
    got2, it2 = pagerank_dev(L, A, DAMPING, 0.0, 12)
    assert it == it2 == 12 and np.array_equal(got.view(np.uint64), got2.view(np.uint64)), "run to run: identical bits"
    want, wit = orc.pagerank(A, DAMPING, 0.0, 12)
    din = max_in_degree(A)
    nsink = int((np.diff(A.p) == 0).sum())
    b = pr_bound(din, nb)
    b_oracle = 8 * (din + nsink + 32) * U
    rel = float(np.max(np.abs(got - want) / want))
    assert wit == 12 and rel <= b + b_oracle, f"rel err {rel} vs {b + b_oracle}"
    assert abs(math.fsum(got.tolist()) - 1.0) <= b


# ------------------------------------------------------------------------------------------ LAGr_ConnectedComponents
def wcc_dev(L, S):
    """(component vector, rounds): the rounds from the launch count -- k_iota_u64, then k_cc_hook + k_cc_jump per round"""
    G = _graph(L, S, 0)
    comp = P()
    l0 = fb.get_stat("launches")
    info = L.LAGr_ConnectedComponents(C.byref(comp), G, None)
    launches = fb.get_stat("launches") - l0
    assert info == 0, f"LAGr_ConnectedComponents returned {info}"
    n = S.nrows
    nv = C.c_uint64(n)
    I, X = np.empty(max(n, 1), np.uint64), np.empty(max(n, 1), np.int64)
    check(L.GrB_Vector_extractTuples_INT64(I.ctypes.data, X.ctypes.data, C.byref(nv), comp))
    assert nv.value == n and np.array_equal(I[:n], np.arange(n))
    L.GrB_Vector_free(C.byref(comp))
    L.LAGraph_Delete(C.byref(G), None)
    return X[:n], (launches - 1) // 2 if n else 0


def bitrev_order(n):
    bits = max(1, (n - 1).bit_length())
    i = np.arange(n, dtype=np.int64)
    r = np.zeros(n, np.int64)
    for b in range(bits):
        r |= ((i >> b) & 1) << (bits - 1 - b)
    return np.argsort(r, kind="stable")


@pytest.mark.gpu
def test_wcc_small_and_degenerate(dev):
    L, _, _ = dev
    rng = np.random.default_rng(4)
    cases = [(0, []), (1, []), (1, [(0, 0)]), (1000, [])]
    a, b = rng.integers(0, 2000, 1500), rng.integers(0, 2000, 1500)
    cases.append((2000, list(zip(a.tolist(), b.tolist()))))
    for n, pairs in cases:
        S = sym_csr(n, [x for x, _ in pairs], [y for _, y in pairs])
        got, rounds = wcc_dev(L, S)
        assert np.array_equal(got, wcc_py(n, pairs)), n
        assert rounds <= 65


@pytest.mark.gpu
def test_wcc_hard_graphs_at_n_big(dev):
    L, _, nb = dev
    ids = np.arange(nb, dtype=np.int64)
    # a path numbered in descending order: one hook round links every vertex below the next, the full chase flattens it, and the
    # second round finds nothing to hook -- exactly two rounds
    got, rounds = wcc_dev(L, sym_csr(nb, ids[1:][::-1], ids[:-1][::-1]))
    assert np.all(got == 0) and rounds == 2, rounds
    o = bitrev_order(nb)
    got, _ = wcc_dev(L, sym_csr(nb, o[:-1], o[1:]))
    assert np.all(got == 0), "bit-reversal path"
    k = np.arange(1, nb, dtype=np.int64)                  # heap layout, node k has id nb - 1 - k: the root has the largest id
    S = sym_csr(nb, nb - 1 - k, nb - 1 - (k - 1) // 2)
    got, _ = wcc_dev(L, S)
    assert np.all(got == 0), "binary tree"
    rng = np.random.default_rng(9)
    hub = nb // 2 + 11
    leaves = rng.choice(nb, 200_001, replace=False)
    leaves = leaves[leaves != hub][:200_000]
    S = sym_csr(nb, np.full(len(leaves), hub), leaves)
    got, _ = wcc_dev(L, S)
    assert np.array_equal(got, orc.wcc(S))


# ------------------------------------------------------------------------------------------ LAGraph_cdlp
def cdlp_dev(L, S, itermax):
    """(labels, rounds): the rounds from the launch count -- k_iota_u64, then k_cdlp_keys + k_cdlp_pick per round"""
    G = _graph(L, S, 0)
    out = P()
    l0 = fb.get_stat("launches")
    assert L.LAGraph_cdlp(C.byref(out), G, itermax, None) == 0
    launches = fb.get_stat("launches") - l0
    n = S.nrows
    nv = C.c_uint64(n)
    I, X = np.empty(max(n, 1), np.uint64), np.empty(max(n, 1), np.int64)
    check(L.GrB_Vector_extractTuples_INT64(I.ctypes.data, X.ctypes.data, C.byref(nv), out))
    assert nv.value == n and np.array_equal(I[:n], np.arange(n))
    L.GrB_Vector_free(C.byref(out))
    L.LAGraph_Delete(C.byref(G), None)
    return X[:n], (launches - 1) // 2 if n else 0


def _cdlp_case(L, n, pairs, itermax):
    S = sym_csr(n, [a for a, _ in pairs], [b for _, b in pairs])
    got, rounds = cdlp_dev(L, S, itermax)
    want, wr = cdlp_py(n, pairs, itermax)
    assert np.array_equal(got, want) and rounds == wr, (n, itermax, rounds, wr)
    return got, rounds


@pytest.mark.gpu
def test_cdlp_known_answers(dev):
    L, _, _ = dev
    for itermax in (1, 2, 3, 4):                           # one edge oscillates and never reaches a fixed point
        got, rounds = _cdlp_case(L, 2, [(0, 1)], itermax)
        assert got.tolist() == ([1, 0] if itermax % 2 else [0, 1]) and rounds == itermax
    a, b = 3, 5                                            # K_{3,5}: the sides swap the labels {0, 3}
    kab = [(i, a + j) for i in range(a) for j in range(b)]
    for itermax in (1, 2, 3):
        got, _ = _cdlp_case(L, a + b, kab, itermax)
        left, right = (a, 0) if itermax % 2 else (0, a)
        assert got.tolist() == [left] * a + [right] * b
    # a 2-2 tie in round 2: vertex 100 sees labels 40, 40 (from 1, 2) and 45, 45 (from 3, 4); the smaller wins
    tie = [(100, 1), (100, 2), (100, 3), (100, 4), (1, 40), (2, 40), (3, 45), (4, 45)]
    got, _ = _cdlp_case(L, 101, tie, 2)
    assert got[100] == 40
    got, _ = _cdlp_case(L, 101, [(7, 60), (7, 9), (5, 5)], 1)
    assert got[7] == 9 and got[5] == 5, "a 1-1 tie takes the smaller label; a self-loop-only vertex keeps its own"
    got, rounds = _cdlp_case(L, 8, [(0, 1), (2, 3)], 0)
    assert got.tolist() == list(range(8)) and rounds == 0
    for n, pairs in ((0, []), (1, []), (1, [(0, 0)])):
        _cdlp_case(L, n, pairs, 3)
    nleaf = 100_000                                        # a hub above its leaves takes the smallest leaf label
    S = sym_csr(nleaf + 1, np.full(nleaf, nleaf), np.arange(nleaf))
    got, rounds = cdlp_dev(L, S, 1)
    want, _ = orc.cdlp(S, 1)
    assert np.array_equal(got, want) and got[nleaf] == 0 and np.all(got[:nleaf] == nleaf) and rounds == 1


@pytest.mark.gpu
def test_cdlp_sort_width_boundary_and_n_big(dev):
    """n = 2^16 and 2^16 + 1 sit on either side of a bits(n) step of the sort's end_bit = 32 + bits(n); N_BIG reaches the second
    grid sweep of k_cdlp_keys and k_cdlp_pick"""
    L, _, nb = dev
    rng = np.random.default_rng(12)
    for n in (1 << 16, (1 << 16) + 1):
        m = 2 * n
        a, b = rng.integers(0, n, m), rng.integers(0, n, m)
        a = np.concatenate([a, np.full(40, n - 1)])        # the last row, the one that needs the top row bit, is long
        b = np.concatenate([b, rng.integers(0, n, 40)])
        S = sym_csr(n, a, b)
        states = cdlp_sorted(S, 5)
        for itermax in (1, 5):
            got, rounds = cdlp_dev(L, S, itermax)
            wr = min(itermax, len(states) - 1)
            assert np.array_equal(got, states[wr]) and rounds == wr, (n, itermax)
    a = np.arange(nb, dtype=np.int64)
    S = sym_csr(nb, np.concatenate([a, a]), rng.integers(0, nb, 2 * nb))
    states = cdlp_sorted(S, 10)
    for itermax in (3, 10):
        got, rounds = cdlp_dev(L, S, itermax)
        wr = min(itermax, len(states) - 1)
        assert rounds == wr and np.array_equal(got, states[wr]), itermax
