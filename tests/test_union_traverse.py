"""Union hops (-[:R1|R2]->): B200_Matrix_union_lmxm and B200_traverse_batch_union, F <- F * U_t (m_t \\ dm_t) u dp_t, exact.
Every case is compared with scipy over the effective operands built on the host (entries and flops, flops of a union hop being
sum_t flops(F*m_t) + flops(F*dp_t)), and with the reference's route: the union built by extract plus set_pattern
(union_by_extract), then B200_traverse_batch over the fresh matrix, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Descriptor, Matrix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    yield
    for k, v in (("bits_mode", -1), ("pull_mode", -1), ("hot_pack", 1), ("csr_push", 1), ("union_accum", 1), ("timing", 0)):
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


def spm(n, pairs):
    pairs = list(set(pairs))
    return sp.csr_matrix((np.ones(len(pairs), np.int64), ([a for a, _ in pairs], [b for _, b in pairs])), shape=(n, n))


def flops(F, n, pairs):
    """flops(F * A): sum over the entries (i, k) of F of the out-degree of k in A"""
    deg = np.bincount(np.array([a for a, _ in set(pairs)], np.int64), minlength=n) if pairs else np.zeros(n, np.int64)
    return int((F @ deg).sum())


def ref_chain(n, src, hops):
    """scipy over the effective operands.  hops: ("union", [(m, dp, dm), ...]) / ("delta", (m, dp, dm)) of host pair lists.
    Returns (dense k x n result, flops)."""
    k = len(src)
    F = sp.csr_matrix((np.ones(k, np.int64), (np.arange(k), src)), shape=(k, n))
    fl = 0
    for kind, ops in hops:
        if kind == "union":
            fl += sum(flops(F, n, m) + flops(F, n, dp or ()) for m, dp, dm in ops)
            A = spm(n, set().union(*[effective(*o) for o in ops]))
            F = sp.csr_matrix(((F @ A) > 0).astype(np.int64))
        else:
            m, dp, dm = ops
            fl += flops(F, n, m) + flops(F, n, dp or ()) + flops(F, n, dm or ())
            Y = ((F @ spm(n, m)).toarray() > 0) & ~((F @ spm(n, dm or ())).toarray() > 0) | ((F @ spm(n, dp or ())).toarray() > 0)
            F = sp.csr_matrix(Y.astype(np.int64))
    return F.toarray() > 0, fl


def union_by_extract(n, dev_ops):
    """Graph::build_relationship_matrix_unrestricted (graph.rs:2520-2550): extract(T_1), then per further type
    set_pattern(<!dm_t> m_t) and set_pattern(dp_t), as a fresh matrix"""
    U = Matrix(n, n, bool)
    m, dp, dm = dev_ops[0]
    U.set_pattern(None, m)
    if dm is not None and dm.nvals():
        U.remove_all(dm)
    if dp is not None and dp.nvals():
        U.set_pattern(None, dp)
    for m, dp, dm in dev_ops[1:]:
        U.set_pattern(dm, m, None if dm is None else Descriptor.C)
        if dp is not None:
            U.set_pattern(None, dp)
    U.wait()
    return U


def run(src, n, dev_hops, fmt=fb.OUT_CSR, cap=None):
    """B200_traverse_batch_union over dev_hops (("union", [(m, dp, dm), ...]) / ("delta", (m, dp, dm))): (dense, flops, nvals)"""
    hs = [[o[0] for o in ops] if kind == "union" else ops[0] for kind, ops in dev_hops]
    ds = [[(o[1], o[2]) for o in ops] if kind == "union" else (ops[1], ops[2]) for kind, ops in dev_hops]
    return traverse(src, n, hs, ds, fmt, cap)


def traverse(src, n, hs, ds, fmt=fb.OUT_CSR, cap=None):
    k, wpr = len(src), (n + 63) // 64
    bits = np.zeros((k, wpr), np.uint64)
    p, j = np.zeros(k + 1, np.uint64), np.zeros(cap if cap is not None else k * n + 1, np.uint32)
    fl, nv, chosen = fb.traverse_batch(src, hs, fmt, out_bitmap=None if fmt == fb.OUT_CSR else bits,
                                       out_p=None if fmt == fb.OUT_BITMAP else p, out_j=None if fmt == fb.OUT_BITMAP else j, deltas=ds)
    out = np.zeros((k, n), bool)
    if chosen == fb.OUT_BITMAP:
        out = np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :n].astype(bool)
    else:
        rows = np.repeat(np.arange(k), np.diff(p.astype(np.int64)))
        out[rows, j[:int(p[-1])].astype(np.int64)] = True
    return out, fl, nv


def via_extract(src, n, dev_hops, fmt=fb.OUT_CSR):
    """the reference's route: every union hop's operand built by union_by_extract, then B200_traverse_batch(_delta)"""
    hs, ds = [], []
    for kind, ops in dev_hops:
        if kind == "union":
            hs.append(union_by_extract(n, ops))
            ds.append((None, None))
        else:
            hs.append(ops[0])
            ds.append((ops[1], ops[2]))
    return traverse(src, n, hs, ds, fmt)


def check(n, hops, dev_hops, src, what="", fmt=fb.OUT_CSR):
    want, wfl = ref_chain(n, src, hops)
    got, fl, nv = run(src, n, dev_hops, fmt)
    assert np.array_equal(got, want), f"{int((got != want).sum())} entries differ {what}"
    assert fl == wfl, f"flops {fl} != {wfl} {what}"
    if nv is not None:
        assert nv == int(want.sum()), what
    ref, _, _ = via_extract(src, n, dev_hops, fmt)
    assert np.array_equal(got, ref), f"differs from union_by_extract {what}"
    return got


def dense_bits(F):
    bits, _ = F.export_bitmap()
    return np.unpackbits(bits.view(np.uint8), axis=1, bitorder="little")[:, :F.ncols()].astype(bool)


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
    """three RMAT operands: 0 and 2 with dirty deltas, 1 clean; operand 0 UINT64 with a BOOL dm; all prepared"""
    fb.init()
    rng = np.random.default_rng(17)
    ops, dev = [], []
    for t in range(3):
        A = orc.rmat_csr(SCALE, 8, 21 + t)
        if t == 1:
            m, dp, dm = random_operand(rng, A, 0, 0, 0, 0, 0)
        else:
            m, dp, dm = random_operand(rng, A, ndel=300, nadd=200, overlap=20, outside=20, both=10)
        ops.append((m, dp, dm))
        dtype = "u64" if t == 0 else bool
        dev.append((to_dev(N, m, dtype).prepare(), to_dev(N, dp, dtype), to_dev(N, dm)))
    deg = np.diff(orc.rmat_csr(SCALE, 8, 21).p)
    src = rng.permutation(N)[:1500]                # sources with and without out-edges
    src[src == np.argmax(deg)] = src[0]
    src[0] = np.argmax(deg)                        # a hub first, so that a 1-row frontier has work
    return ops, dev, src


@pytest.mark.parametrize("pull_mode", [-1, 0, 1])
@pytest.mark.parametrize("nops", [2, 3])
@pytest.mark.parametrize("nsrc", [1, 64, 100, 200, 512, 1024])
def test_frontier_grid(world, nsrc, nops, pull_mode):
    """W = 1, 1, 2, 4, 8, 16; 2 and 3 operands; every pull mode; hot-set packing on and off; one and two union hops"""
    ops, dev, src = world
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", pull_mode)
    order = [1, 0, 2][:nops] if nops == 3 else [1, 0]        # a clean operand first: the dirty one is moved ahead of it
    u = [ops[t] for t in order]
    du = [dev[t] for t in order]
    for hot in (0, 1):
        fb.set_option("hot_pack", hot)
        for nh in (1, 2):
            check(N, [("union", u)] * nh, [("union", du)] * nh, src[:nsrc],
                  f"(nsrc={nsrc} nops={nops} pull={pull_mode} hot={hot} hops={nh})", fmt=fb.OUT_BITMAP if nh == 2 else fb.OUT_CSR)


@pytest.mark.parametrize("nsrc", [64, 1500])
def test_row_wise_fallback(world, nsrc):
    """bits_mode 0, and more than 1024 rows with bits_mode -1: the union is materialised once per call for GrB_mxm"""
    ops, dev, src = world
    for mode in (0, -1):
        fb.set_option("bits_mode", mode)
        for nops in (2, 3):
            check(N, [("union", ops[:nops])] * 2, [("union", dev[:nops])] * 2, src[:nsrc], f"(bits_mode={mode} nsrc={nsrc} nops={nops})")


def test_accumulation_off_gives_the_same(world):
    """union_accum = 0 (a bit-matrix per operand plus an OR pass) and the accumulating product agree, bit for bit and in flops"""
    ops, dev, src = world
    fb.set_option("bits_mode", 1)
    for nsrc in (64, 1024):
        for pull in (-1, 0, 1):
            fb.set_option("pull_mode", pull)
            got = {}
            for acc in (1, 0):
                fb.set_option("union_accum", acc)
                got[acc] = run(src[:nsrc], N, [("union", dev)] * 2)
            assert np.array_equal(got[0][0], got[1][0]) and got[0][1] == got[1][1], f"(nsrc={nsrc} pull={pull})"


def test_hop1_from_csr_and_accumulating_kernels(world):
    """hop 1 of a small CSR frontier keeps the CSR push for every operand (path 7, "bits_push_acc" for the clean ones); a dense
    frontier pulls and its clean operands OR into the product ("bits_pull_acc")"""
    ops, dev, src = world
    fb.set_option("bits_mode", 1)
    fb.set_option("timing", 1)
    stat = lambda name: (lambda ms, nl, by: (lib().B200_kernel_stats(name, C.byref(ms), C.byref(nl), C.byref(by)), nl.value)[1])(
        C.c_double(), U64(), U64())
    u, du = [ops[1], ops[0], ops[2]], [dev[1], dev[0], dev[2]]
    want, _ = ref_chain(N, src[:40], [("union", u)])
    F = Matrix(40, N, bool)
    F.build(np.arange(40), src[:40])
    fb.reset_stats()
    F.union_lmxm([d[0] for d in du], [(d[1], d[2]) for d in du])
    assert fb.get_stat("last_path") == 7, "hop 1 did not push from the CSR frontier"
    assert stat(b"bits_push_acc") >= 1
    assert np.array_equal(dense_bits(F), want)
    fb.set_option("pull_mode", 1)
    want2, _ = ref_chain(N, src[:1024], [("union", u)] * 2)
    F = Matrix(1024, N, bool)
    F.build(np.arange(1024), src[:1024])
    F.union_lmxm([d[0] for d in du], [(d[1], d[2]) for d in du])
    fb.reset_stats()
    F.union_lmxm([d[0] for d in du], [(d[1], d[2]) for d in du])
    assert fb.get_stat("last_path") == 3 and stat(b"bits_pull_acc") >= 1
    assert np.array_equal(dense_bits(F), want2)


def test_edge_cases():
    """m_1 entries in dm_2 survive; a dp_2 entry on a pair deleted in type 1; overlapping and non-subset deltas; two operands with
    a non-empty dm; NULL and empty deltas; UINT64 operands with a BOOL dm"""
    n = 16
    m1 = [(0, 1), (1, 2), (2, 3), (3, 3), (4, 5), (5, 6), (0, 7)]
    m2 = [(0, 8), (8, 9), (1, 10), (4, 11)]
    cases = [
        ((m1, [], []), (m2, [], [(0, 1), (1, 2)])),                      # dm_2 holds m_1 entries: they survive
        ((m1, [], [(0, 1), (1, 2)]), (m2, [(0, 1)], [])),                # dp_2 re-adds a pair type 1 deleted; (1, 2) stays gone
        ((m1, [(1, 2), (9, 9)], [(1, 2), (0, 9)]), (m2, [(0, 9)], [(8, 9), (0, 12)])),   # overlapping and non-subset deltas
        ((m1, [], [(4, 5), (0, 7)]), (m2, [], [(0, 8), (4, 11)])),       # two operands with a non-empty dm
        ((m1, [], []), (m2, [], [])),                                    # empty deltas
    ]
    src = [0, 4, 3, 11, 8]
    for mode in (1, 0):
        fb.set_option("bits_mode", mode)
        for pull in (-1, 0, 1):
            fb.set_option("pull_mode", pull)
            for case in cases:
                dev = [(to_dev(n, m, "u64").prepare(), to_dev(n, dp, "u64"), to_dev(n, dm)) for m, dp, dm in case]
                for nh in (1, 2, 3):
                    check(n, [("union", list(case))] * nh, [("union", dev)] * nh, src, f"(mode={mode} pull={pull} {case} hops={nh})")
            M1, M2 = to_dev(n, m1).prepare(), to_dev(n, m2).prepare()
            check(n, [("union", [(m1, [], []), (m2, [], [])])], [("union", [(M1, None, None), (M2, None, None)])], src, "(NULL deltas)")
            check(n, [("union", [(m1, [], []), (m2, [], [(0, 1)])])],
                  [("union", [(M1, None, None), (M2, None, to_dev(n, [(0, 1)]))])], src, "(a NULL and a dirty operand)")
    # the first row's dm survives: (0, 1) of m_1 is in dm_2, and 1 is reached
    got = check(n, [("union", list(cases[0]))], [("union", [(to_dev(n, m, "u64").prepare(), to_dev(n, dp, "u64"), to_dev(n, dm))
                                                            for m, dp, dm in cases[0]])], [0])
    assert got[0, 1] and got[0, 8]


def test_one_operand_union_hop_is_exact_where_the_delta_hop_over_masks():
    """s->a, s->b, a->c, b->c with a->c deleted: the one-operand union hop keeps c (it is reached through b), the delta hop over
    the same operand drops it -- the hop kind is stated, not inferred from the operand count"""
    n, s, a, b, c = 8, 0, 1, 2, 3
    m, dm = [(s, a), (s, b), (a, c), (b, c)], [(a, c)]
    M, DM = to_dev(n, m), to_dev(n, dm)
    for mode in (1, 0):
        fb.set_option("bits_mode", mode)
        hops_u = [("delta", (m, [], [])), ("union", [(m, [], dm)])]
        got = check(n, hops_u, [("delta", (M, None, None)), ("union", [(M, None, DM)])], [s], f"(bits_mode={mode})")
        assert got[0, c]
        got = check(n, [("delta", (m, [], [])), ("delta", (m, [], dm))], [("delta", (M, None, None)), ("delta", (M, None, DM))],
                    [s], f"(bits_mode={mode})")
        assert not got[0, c]
        F = Matrix(1, n, bool)
        F.build([0], [s])
        F.union_lmxm([M], [(None, None)])
        F.union_lmxm([M], [(None, DM)])
        F.wait()
        assert F.contains(0, c)


@pytest.mark.parametrize("nsrc", [64, 300])
def test_mixed_chain_formats_and_space(world, nsrc):
    """a delta hop, a union hop, a diagonal label hop: CSR, bitmap and automatic hand-off, and GrB_INSUFFICIENT_SPACE"""
    ops, dev, src = world
    rng = np.random.default_rng(5)
    lab = sorted(rng.choice(N, N // 3, replace=False).tolist())
    L = [(v, v) for v in lab]
    DL = to_dev(N, L).prepare()
    hops = [("delta", ops[0]), ("union", ops[1:3]), ("delta", (L, [], []))]
    dh = [("delta", dev[0]), ("union", dev[1:3]), ("delta", (DL, None, None))]
    for mode in (1, -1, 0):
        fb.set_option("bits_mode", mode)
        for fmt in (fb.OUT_CSR, fb.OUT_BITMAP, fb.OUT_AUTO):
            check(N, hops, dh, src[:nsrc], f"(mode={mode} fmt={fmt})", fmt=fmt)
        want, _ = ref_chain(N, src[:nsrc], hops)
        with pytest.raises(BufferError):
            run(src[:nsrc], N, dh, fb.OUT_CSR, cap=int(want.sum()) - 1)


def test_multi_operand_reach_unchanged(world):
    """B200_reach_batch_delta over 2 and 3 operands after the shared union_product: the scipy level loop, accumulating or not"""
    ops, dev, src = world
    fb.set_option("bits_mode", 1)

    def ref_reach(n, ops, src, max_hops):
        A = spm(n, set().union(*[effective(*o) for o in ops]))
        k = len(src)
        F = sp.csr_matrix((np.ones(k, np.int64), (np.arange(k), src)), shape=(k, n))
        R = np.zeros((k, n), bool)
        for _ in range(max_hops):
            Y = ((F @ A).toarray() > 0) & ~R
            if not Y.any():
                break
            R |= Y
            F = sp.csr_matrix(Y.astype(np.int64))
        return R

    for acc in (1, 0):
        fb.set_option("union_accum", acc)
        for nops in (2, 3):
            for k in (64, 1024):
                R, _ = fb.reach_batch(src[:k], [d[0] for d in dev[:nops]], 3, False, deltas=[(d[1], d[2]) for d in dev[:nops]])
                R.wait()
                p, j, _ = R.export_csr()
                got = np.zeros((k, N), bool)
                got[np.repeat(np.arange(k), np.diff(p.astype(np.int64))), j.astype(np.int64)] = True
                assert np.array_equal(got, ref_reach(N, ops[:nops], src[:k], 3)), f"(acc={acc} nops={nops} k={k})"


def test_host_mirror_union_hop():
    """expand_batch over a multi-type TraversalMatrix, per hop and coalesced, equals the union_by_extract route"""
    L = C.CDLL(os.path.join(ROOT, "falkordb_b200", "libfdbhost.so"))
    L.fdbh_run_test.argtypes = [C.c_char_p]
    L.fdbh_last_message.restype = C.c_char_p
    assert L.fdbh_run_test(b"union_traverse_over_tensor_types") == 0, L.fdbh_last_message().decode()
