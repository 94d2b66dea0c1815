"""The CSR push's gate (csr_push.cu: csr_push_wins) and its relabelled operand (PullTables::ap).  A CSR frontier pushes straight from
its entries when flops * 4 <= nnz(A), or when the bit-matrix hop would push too (edges * 4 <= nnz(A), edges = the out-degrees
summed over the DISTINCT columns of F) and the duplicate flops it would merge stay under n * W / 2.  Frontiers here are built with
a known duplication: edges from a pool of vertices, flops - edges from placing some of them in further rows.  Through a prepared
operand the push reads A.col_idx already relabelled to the hot-set order, a table that has to follow every change of the operand.
(tests/test_zz4_ordered_frontier.py predicts the path from flops * 4 <= nnz(A) alone, which holds for its cases only.)"""
import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix
from test_gpu_parity import to_dev, assert_same
from test_delta_traverse import deltas

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    yield
    for k, v in (("bits_mode", -1), ("pull_mode", -1), ("csr_push", 1), ("perm_push", 1), ("hot_pack", 1)):
        fb.set_option(k, v)


def dup_frontier(A, nsrc, share, extra, seed):
    """nsrc rows over a pool of random vertices whose out-degrees sum to about share * nnz(A), each in one random row; then pool
    vertices are placed in further rows (row + 1, row + 2, ... for successive layers) until their degrees add about
    extra * nnz(A) flops, so flops - edges ~ extra * nnz(A) while edges ~ share * nnz(A)"""
    rng = np.random.default_rng(seed)
    deg = np.diff(A.p).astype(np.int64)
    live = rng.permutation(np.nonzero(deg)[0])
    pool = live[:np.searchsorted(np.cumsum(deg[live]), share * A.nnz) + 1]
    row = rng.integers(0, nsrc, len(pool))
    rows, cols = [row], [pool]
    left, layer = extra * A.nnz, 1
    cs = np.cumsum(deg[pool])
    while left > 0:
        m = min(len(pool), int(np.searchsorted(cs, left)) + 1)
        rows.append((row[:m] + layer) % nsrc)
        cols.append(pool[:m])
        left -= cs[m - 1]
        layer += 1
    return orc.build_matrix(nsrc, A.nrows, np.concatenate(rows), np.concatenate(cols))


def gate(F, A):
    """(flops, edges, W, whether csr_push_wins takes it) computed on the host"""
    deg = np.diff(A.p).astype(np.int64)
    fl, ed = int(deg[F.j].sum()), int(deg[np.unique(F.j)].sum())
    W = 1
    while W * 64 < F.nrows:
        W *= 2
    take = fl * 4 <= A.nnz or (ed * 4 <= A.nnz and (fl - ed) * 2 <= A.nrows * W)
    return fl, ed, W, take


def hop(F0, dA, **opts):
    """F0 * dA from F0's CSR form under the given options; returns (result, path, flops)"""
    fb.set_option("bits_mode", 1)
    for k, v in opts.items():
        fb.set_option(k, v)
    try:
        F = to_dev(F0, bool)
        F.lmxm(dA)
        path, fl = fb.get_stat("last_path"), fb.get_stat("last_flops")
        F.wait()
        return F, path, fl
    finally:
        for k, v in (("csr_push", 1), ("pull_mode", -1), ("perm_push", 1)):
            fb.set_option(k, v)


@pytest.mark.parametrize("nsrc,share,extra", [(64, 0.23, 0.025), (512, 0.12, 0.2), (1024, 0.12, 0.4)])   # W = 1, 8, 16
def test_repeated_vertices_push_from_csr_entries(nsrc, share, extra):
    """flops * 4 > nnz(A), edges * 4 <= nnz(A), flops - edges <= n * W / 2: path 7, the same product as the bit-matrix push, the
    pull, the push through pperm without the relabelled table, the natural-order push and the oracle"""
    A = orc.rmat_csr(14, 16, 5)
    F0 = dup_frontier(A, nsrc, share, extra, nsrc)
    fl, ed, W, take = gate(F0, A)
    assert fl * 4 > A.nnz and ed * 4 <= A.nnz and take, (fl, ed, W, A.nnz)
    want = orc.mxm(F0, A)
    dA = to_dev(A, bool).prepare(True)
    for opts, path in (({}, 7), ({"csr_push": 0}, 2), ({"pull_mode": 1}, 3), ({"perm_push": 0}, 7)):
        F, got_path, got_fl = hop(F0, dA, **opts)
        assert got_path == path, (opts, got_path)
        assert got_fl == fl, f"{opts}: last_flops {got_fl} != mxm flops {fl}"
        assert_same(F, want, f"nsrc={nsrc} {opts}")
    fb.set_option("perm_push", 0)                     # tables without the relabelled col_idx: the push reads pperm[col]
    dB = to_dev(A, bool).prepare(True)
    fb.set_option("perm_push", 1)
    F, got_path, _ = hop(F0, dB)
    assert got_path == 7
    assert_same(F, want, f"nsrc={nsrc}: push through pperm")


@pytest.mark.parametrize("nsrc,share,extra", [(512, 0.12, 0.5), (1024, 0.2, 0.75)])
def test_frontier_that_repeats_hubs_takes_the_bit_matrix_push(nsrc, share, extra):
    """flops - edges > n * W / 2: the bit-matrix hop merges the repeats into one RED per word, so the CSR push declines (path 2);
    csr_push = 2 forces it, with the same product"""
    A = orc.rmat_csr(14, 16, 6)
    F0 = dup_frontier(A, nsrc, share, extra, 1)
    fl, ed, W, take = gate(F0, A)
    assert ed * 4 <= A.nnz and not take and F0.nnz <= 1 << 20, (fl, ed, W)
    want = orc.mxm(F0, A)
    dA = to_dev(A, bool).prepare(True)
    F, path, got_fl = hop(F0, dA)
    assert path == 2 and got_fl == fl
    assert_same(F, want, "declined push")
    F, path, got_fl = hop(F0, dA, csr_push=2)
    assert path == 7 and got_fl == fl
    assert_same(F, want, "forced push")


def test_wide_frontier_still_pulls():
    """edges * 4 > nnz(A): the CSR push declines and the pull takes the hop"""
    A = orc.rmat_csr(14, 16, 6)
    F0 = dup_frontier(A, 64, 0.5, 0.3, 1)
    fl, ed, _, take = gate(F0, A)
    assert ed * 4 > A.nnz and not take and F0.nnz <= 1 << 20        # small enough to be probed
    dA = to_dev(A, bool).prepare(True)
    F, path, got_fl = hop(F0, dA)
    assert path == 3 and got_fl == fl
    assert_same(F, orc.mxm(F0, A), "declined push")


@pytest.mark.parametrize("nsrc", [512, 1024])
def test_ordered_pull_follows_the_push(nsrc):
    """the push through a prepared operand leaves Y in its hot-set order and the next hop pulls from it; perm_push 0 (natural
    order, no relabelled table) gives the same chain"""
    A = orc.rmat_csr(14, 16, 7)
    F0 = dup_frontier(A, nsrc, 0.15, 0.2, 2 * nsrc)
    fl, ed, _, take = gate(F0, A)
    assert fl * 4 > A.nnz and take
    want2 = orc.mxm(F0, A)
    want3 = orc.mxm(want2, A)
    dA = to_dev(A, bool).prepare(True)
    fb.set_option("bits_mode", 1)
    for perm in (1, 0):
        fb.set_option("perm_push", perm)
        F = to_dev(F0, bool)
        F.lmxm(dA)
        assert fb.get_stat("last_path") == 7
        assert F.nvals() == want2.nnz
        G = F.dup()
        G.wait()
        assert_same(G, want2, f"pushed hop, perm_push={perm}")
        F.lmxm(dA)
        assert fb.get_stat("last_path") == 3
        assert_same(F, want3, f"pull after the push, perm_push={perm}")


def rewire(dA, have, ks, rng, n):
    """drop one out-edge of each vertex in ks and add an edge to a fresh column, on the device matrix and in the host pair set"""
    for k in ks.tolist():
        j = min(t for s, t in have if s == k)
        dA.remove(k, j)
        have.discard((k, j))
        t = int(rng.integers(0, n))
        while (k, t) in have or t == k:
            t = int(rng.integers(0, n))
        dA.set(k, t)
        have.add((k, t))
    dA.wait()
    r = np.array([a for a, _ in have], np.uint64)
    c = np.array([b for _, b in have], np.uint64)
    return orc.build_matrix(n, n, r, c)


def test_relabelled_operand_follows_the_matrix():
    """the relabelled col_idx is rebuilt with the pull tables after the operand changes, by the first pull that builds them and
    by prepare, and it is added when hot_pack is turned on after the tables were built without it"""
    A = orc.rmat_csr(13, 16, 8)
    n = A.nrows
    F0 = dup_frontier(A, 256, 0.2, 0.08, 3)
    fl, ed, _, take = gate(F0, A)
    assert fl * 4 > A.nnz and take
    dA = to_dev(A, bool).prepare(True)
    F, path, _ = hop(F0, dA)
    assert path == 7
    assert_same(F, orc.mxm(F0, A), "before the change")
    rng = np.random.default_rng(4)
    have = A.tuple_set()
    cols = np.unique(F0.j)

    # change 1: the first pull rebuilds the mirror and the tables lazily
    A1 = rewire(dA, have, rng.choice(cols, 50, replace=False), rng, n)
    want = orc.mxm(F0, A1)
    G = to_dev(F0, bool)
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", 1)
    G.lmxm(dA)
    assert fb.get_stat("last_path") == 3
    assert_same(G, want, "pull after change 1")
    fb.set_option("pull_mode", -1)
    F, path, _ = hop(F0, dA)
    assert path == 7
    assert_same(F, want, "push after the tables were rebuilt by a pull")

    # change 2: prepare rebuilds them, with no pull in between
    A2 = rewire(dA, have, rng.choice(cols, 50, replace=False), rng, n)
    want = orc.mxm(F0, A2)
    dA.prepare(True)
    F, path, _ = hop(F0, dA)
    assert path == 7
    assert_same(F, want, "push after change 2 and prepare")

    fb.set_option("hot_pack", 0)                      # tables without the order, then the order added by a later pull
    dB = to_dev(A2, bool).prepare(True)
    F, path, _ = hop(F0, dB)
    assert path == 7
    assert_same(F, want, "push without hot-set order")
    fb.set_option("hot_pack", 1)
    F, path, _ = hop(F0, dB, pull_mode=1)
    assert path == 3
    F = to_dev(F0, bool)
    fb.set_option("bits_mode", 1)
    F.lmxm(dB)
    assert fb.get_stat("last_path") == 7
    F.lmxm(dB)
    assert fb.get_stat("last_path") == 3
    assert_same(F, orc.mxm(want, A2), "push through the table added later, then the ordered pull")


@pytest.mark.parametrize("nsrc", [512, 1024])
def test_dirty_hop_from_csr_through_the_relabelled_operand(nsrc):
    """delta_lmxm with Δ+ and Δ−: the base push reads the relabelled col_idx, the delta pushes go through pperm; both land in
    the same order, and the next dirty hop pulls from it"""
    rng = np.random.default_rng(nsrc)
    A = orc.rmat_csr(14, 16, 9)
    dp, dm = deltas(rng, A, 3000, 3000, overlap=30, outside=30)
    F0 = dup_frontier(A, nsrc, 0.15, 0.2, nsrc + 1)
    fl, ed, _, take = gate(F0, A)
    assert fl * 4 > A.nnz and take
    dA, dpd, dmd = to_dev(A, bool).prepare(True), to_dev(dp, bool), to_dev(dm, bool)
    fb.set_option("bits_mode", 1)
    F, C_ = to_dev(F0, bool), to_dev(F0, bool)
    want = F0
    for h, pm in enumerate((-1, 1)):
        fb.set_option("pull_mode", pm)
        want = orc.delta_lmxm(want, A, dp, dm)
        F.delta_lmxm_fused(dA, dpd, dmd)
        assert fb.get_stat("last_path") == (7, 3)[h]
        C_.delta_lmxm(dA, dpd, dmd)
        assert_same(F, want, f"fused dirty hop {h}")
        assert_same(C_, want, f"composed dirty hop {h}")
