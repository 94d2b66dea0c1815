"""The sliced CSR push (csr_push.cu: csr_push_sliced).  Through a prepared operand whose relabelled col_idx (PullTables::ap) has every
row ascending by position, the push cuts the positions into destination slices and issues the same REDs slice by slice.  Nothing
about the product may depend on the slice count, so chains run with push_slices forced to 1, 3, 7 and more slices than vertices
and are compared with the oracle by digest and by exported CSR; the routes that never slice (accumulating union hops, the delta
pushes of a dirty hop, perm_push off) must give what push_slices = 0 gives."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix

SCALE = 12
N = 1 << SCALE
OPTS = (("bits_mode", -1), ("pull_mode", -1), ("csr_push", 1), ("perm_push", 1), ("push_slices", -1), ("timing", 0))


@pytest.fixture
def defaults():
    fb.init()
    yield
    for k, v in OPTS:
        fb.set_option(k, v)


def graph(seed):
    """RMAT-12 with the out-edges of a few vertices removed, so that some frontier columns have an empty row of A"""
    A = orc.rmat_csr(SCALE, 16, seed)
    deg = np.diff(A.p).astype(np.int64)
    rows = np.repeat(np.arange(N), deg)
    sinks = np.nonzero((deg > 0) & (deg < 4))[0][:8]
    keep = ~np.isin(rows, sinks)
    return orc.build_matrix(N, N, rows[keep], A.j[keep].astype(np.int64)), sinks


def frontier(A, sinks, nsrc, seed, per_row=3):
    """every third row empty; the two largest hubs in a quarter of the rows (repeated columns); the sinks; random vertices"""
    rng = np.random.default_rng(seed)
    deg = np.diff(A.p).astype(np.int64)
    hubs = np.argsort(-deg)[:2]
    rows, cols = [], []
    for i in range(nsrc):
        if i % 3 == 2:
            continue
        c = set(rng.integers(0, N, per_row).tolist())
        if i % 4 == 0:
            c.update(hubs.tolist())
        if i % 16 == 1:
            c.add(int(sinks[i % len(sinks)]))
        rows += [i] * len(c)
        cols += sorted(c)
    return orc.build_matrix(nsrc, N, np.array(rows), np.array(cols)), hubs


def to_dev(c):
    return Matrix.import_csr(c.nrows, c.ncols, c.p.astype(np.uint64), c.j, None, bool)


def same(dev, want, what):
    p, j, _ = dev.export_csr()
    assert np.array_equal(p, want.p) and np.array_equal(j, want.j), f"{what}: the exported CSR differs"
    assert np.array_equal(dev.digest(), orc.digest(want)), f"{what}: the digest differs"


def push_bytes():
    ms, n, b = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    assert fb._lib.lib().B200_kernel_stats(b"bits_push", C.byref(ms), C.byref(n), C.byref(b)) == 0
    return b.value


def rows_are_sorted_permutations(p, j, ap, pperm):
    """every row of ap ascending, and the same multiset as the row of j sent through pperm"""
    rid = np.repeat(np.arange(len(p) - 1), np.diff(p.astype(np.int64)))
    inside = rid[1:] == rid[:-1]
    if np.any(inside & (ap[1:].astype(np.int64) < ap[:-1].astype(np.int64))):
        return False
    want = pperm[j]
    order = np.lexsort((want, rid))
    return bool(np.array_equal(want[order], ap))


def test_row_check_tells_sorted_permutations_apart():
    """the checker itself, on the host: a relabelled matrix with sorted rows passes; an unsorted row, a changed entry and an entry
    moved to the next row do not"""
    rng = np.random.default_rng(0)
    n = 50
    deg = rng.integers(0, 6, n)
    deg[7] = 0
    p = np.concatenate(([0], np.cumsum(deg))).astype(np.uint64)
    j = np.concatenate([np.sort(rng.choice(n, d, replace=False)) for d in deg]).astype(np.uint32)
    pperm = rng.permutation(n).astype(np.uint32)
    ap = np.concatenate([np.sort(pperm[j[int(p[r]):int(p[r + 1])]]) for r in range(n)]).astype(np.uint32)
    assert rows_are_sorted_permutations(p, j, ap, pperm)
    r = int(np.argmax(deg))
    a, b = int(p[r]), int(p[r + 1])
    bad = ap.copy()
    bad[a:b] = bad[a:b][::-1]
    assert not rows_are_sorted_permutations(p, j, bad, pperm)
    bad = ap.copy()
    bad[a] = (set(range(n)) - set(ap[a:b].tolist())).pop()
    bad[a:b] = np.sort(bad[a:b])
    assert not rows_are_sorted_permutations(p, j, bad, pperm)
    assert not rows_are_sorted_permutations(p, j, np.sort(ap), pperm)       # sorted across rows: rows lose their own entries


@pytest.mark.gpu
def test_sorted_operand_is_a_row_permutation_of_the_relabelled_matrix(defaults):
    A, _ = graph(3)
    dA = to_dev(A).prepare(True)
    ap, pperm, srt = dA.push_operand()
    assert srt and np.array_equal(np.sort(pperm), np.arange(N))
    assert rows_are_sorted_permutations(A.p, A.j, ap, pperm)
    fb.set_option("push_slices", 0)             # tables built with slicing off keep the entry order, and say so
    dB = to_dev(A).prepare(True)
    ap0, pperm0, srt0 = dB.push_operand()
    assert not srt0 and np.array_equal(pperm0, pperm) and np.array_equal(ap0, pperm[A.j])


@pytest.mark.gpu
@pytest.mark.parametrize("nsrc", [64, 512, 1024])                # W = 1, 8, 16
@pytest.mark.parametrize("slices", [1, 3, 7, N + 5])
def test_chain_is_the_oracle_chain_at_any_slice_count(defaults, nsrc, slices):
    A, sinks = graph(5)
    F0, hubs = frontier(A, sinks, nsrc, nsrc + slices, per_row=1 if slices > N else 3)
    dA = to_dev(A).prepare(True)
    ap, _, srt = dA.push_operand()
    assert srt
    if slices in (3, 7):                        # the largest hub has entries in every slice
        S = -(-N // slices)
        hub = ap[int(A.p[hubs[0]]):int(A.p[hubs[0] + 1])]
        assert len(np.unique(hub // S)) == slices
    assert (slices if slices <= N else N) * F0.nnz <= 1 << 24     # below the bound where the push stops slicing
    fb.set_option("bits_mode", 1)
    fb.set_option("csr_push", 2)                # the CSR push whatever the frontier's size
    fb.set_option("timing", 1)
    got = {}
    for ps in (0, slices):
        fb.set_option("push_slices", ps)
        F = to_dev(F0)
        want = F0
        b0 = push_bytes()
        for hop in range(3):
            fb.set_option("csr_push", 2 if hop == 0 else 1)
            F.lmxm(dA)
            if hop == 0:                        # the frontier is a CSR only before its first hop
                assert fb.get_stat("last_path") == 7
                got[ps] = push_bytes() - b0
            want = orc.mxm(want, A)
            G = F.dup()
            G.wait()
            same(G, want, f"hop {hop + 1}, push_slices={ps}")
    # the sliced route accounts 32 bytes per (entry, slice) for its sub-entry table on top of the entry-order push's bytes
    assert got[slices] - got[0] == 32 * F0.nnz * min(slices, N)


@pytest.mark.gpu
@pytest.mark.parametrize("nsrc", [64, 512])
def test_routes_that_never_slice_match_push_slices_off(defaults, nsrc):
    """the accumulating push of a union hop, a dirty hop's delta pushes and the push without the relabelled order"""
    A, sinks = graph(7)
    B = orc.rmat_csr(SCALE, 4, 8)
    rng = np.random.default_rng(nsrc)
    pick = rng.choice(A.nnz, 300, replace=False)
    rows = np.repeat(np.arange(N), np.diff(A.p).astype(np.int64))
    dm = orc.build_matrix(N, N, rows[pick], A.j[pick].astype(np.int64))
    dp = orc.build_matrix(N, N, rng.integers(0, N, 300), rng.integers(0, N, 300))
    F0, _ = frontier(A, sinks, nsrc, nsrc)
    dA, dB, dpd, dmd = to_dev(A).prepare(True), to_dev(B).prepare(True), to_dev(dp), to_dev(dm)
    fb.set_option("bits_mode", 1)
    fb.set_option("csr_push", 2)

    def run(ps, what):
        fb.set_option("push_slices", ps)
        fb.set_option("perm_push", 0 if what == "natural" else 1)
        F = to_dev(F0)
        if what == "union":
            F.union_lmxm([dA, dB])
        elif what == "dirty":
            F.delta_lmxm_fused(dA, dpd, dmd)
        else:
            F.lmxm(dA)
        F.lmxm(dA)
        F.wait()
        return F.export_csr()[:2], tuple(F.digest())

    for what in ("union", "dirty", "natural"):
        (p0, j0), d0 = run(0, what)
        for ps in (-1, 3):
            (p1, j1), d1 = run(ps, what)
            assert np.array_equal(p0, p1) and np.array_equal(j0, j1) and d0 == d1, f"{what}, push_slices={ps}"
    fb.set_option("perm_push", 1)
    fb.set_option("push_slices", 3)
    F = to_dev(F0)
    F.delta_lmxm_fused(dA, dpd, dmd)
    F.wait()
    same(F, orc.delta_lmxm(F0, A, dp, dm), "dirty hop whose base push is sliced")
