"""The pull kernels under their L2 cache policies (bits_hop.cu: k_pull_small, k_pull_seg, PullHints).  A policy only says how long a
line stays in the L2, so no product may depend on it: every instantiation -- W = 1 ... 16, plain and accumulating, with and
without early exit -- runs with hints off and on, with an evict_last prefix of nothing, of part of the gather source and of more
than all of it, and must give the oracle's product bit for bit.  The graph has small rows, mid rows and rows of A' long enough to
be cut into segments that merge with RED.OR."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix

SCALE = 14
N = 1 << SCALE
LONG_ROW = 4096
OPTS = (("bits_mode", -1), ("pull_mode", -1), ("hints", -1), ("hint_streams", -1), ("hot_bytes", -1), ("early_exit", 1),
        ("timing", 0))
# (hints, hint_streams, hot_bytes); hot_bytes = 1 << 40 is more than any gather source here and is cut to its size
POLICIES = [(0, 1, -1), (1, 1, 0), (1, 1, 4096), (1, 0, 100_000), (1, 1, 1 << 40), (1, -1, -1), (-1, -1, -1)]


@pytest.fixture
def defaults():
    fb.init()
    yield
    for k, v in OPTS:
        fb.set_option(k, v)


def graph():
    """RMAT-14 plus two columns of in-degree above LONG_ROW (rows of A' cut into 2 and 3 segments)"""
    A = orc.rmat_csr(SCALE, 4, 11)
    rows = np.repeat(np.arange(N), np.diff(A.p).astype(np.int64))
    cols = A.j.astype(np.int64)
    rng = np.random.default_rng(1)
    extra_r = np.concatenate([rng.choice(N, LONG_ROW + 900, replace=False), rng.choice(N, 2 * LONG_ROW + 7, replace=False)])
    extra_c = np.concatenate([np.full(LONG_ROW + 900, 5), np.full(2 * LONG_ROW + 7, 9)])
    A = orc.build_matrix(N, N, np.concatenate([rows, extra_r]), np.concatenate([cols, extra_c]))
    indeg = np.bincount(A.j.astype(np.int64), minlength=N)
    assert indeg.max() > 2 * LONG_ROW and np.any((indeg > 8) & (indeg <= LONG_ROW)) and np.any((indeg > 0) & (indeg <= 8))
    return A


def frontier(nsrc, seed):
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(nsrc), 2)
    return orc.build_matrix(nsrc, N, rows, rng.integers(0, N, 2 * nsrc))


def to_dev(c):
    return Matrix.import_csr(c.nrows, c.ncols, c.p.astype(np.uint64), c.j, None, bool)


def launches(name):
    ms, n, b = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    return n.value if fb._lib.lib().B200_kernel_stats(name, C.byref(ms), C.byref(n), C.byref(b)) == 0 else 0


def same(dev, want, what):
    dev.wait()
    p, j, _ = dev.export_csr()
    assert np.array_equal(p, want.p) and np.array_equal(j, want.j), f"{what}: the exported CSR differs"
    assert np.array_equal(dev.digest(), orc.digest(want)), f"{what}: the digest differs"


def set_policy(hints, streams, hot, early):
    fb.set_option("hints", hints)
    fb.set_option("hint_streams", streams)
    fb.set_option("hot_bytes", hot)
    fb.set_option("early_exit", early)


@pytest.mark.gpu
@pytest.mark.parametrize("nsrc", [64, 128, 256, 512, 1024])          # W = 1, 2, 4, 8, 16
def test_pull_is_the_oracle_under_every_policy(defaults, nsrc):
    A = graph()
    F0 = frontier(nsrc, nsrc)
    want1 = orc.mxm(F0, A)
    want2 = orc.mxm(want1, A)
    dA = to_dev(A).prepare(True)
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", 1)
    fb.set_option("timing", 1)
    for pol in POLICIES:
        for early in (0, 2):
            set_policy(*pol, early)
            what = f"hints/streams/hot_bytes {pol}, early_exit {early}"
            F = to_dev(F0)
            F.lmxm(dA)                          # from a CSR: the bit-matrix is gathered through the packed copy
            G = F.dup()
            same(G, want1, f"hop 1, {what}")
            n0 = launches(b"bits_pull")
            F.lmxm(dA)                          # from a bit-matrix
            assert fb.get_stat("last_path") == 3 and launches(b"bits_pull") > n0, f"hop 2 did not pull, {what}"
            same(F, want2, f"hop 2, {what}")


@pytest.mark.gpu
@pytest.mark.parametrize("nsrc", [64, 512, 1024])
def test_accumulating_union_pull_is_the_oracle_under_every_policy(defaults, nsrc):
    A = graph()
    B = orc.rmat_csr(SCALE, 4, 12)
    F0 = frontier(nsrc, nsrc + 1)
    dA, dB = to_dev(A).prepare(True), to_dev(B).prepare(True)
    want1 = orc.mxm(F0, A)
    want2 = orc.ewise_add(orc.mxm(want1, A), orc.mxm(want1, B))
    fb.set_option("bits_mode", 1)
    fb.set_option("pull_mode", 1)
    fb.set_option("timing", 1)
    for pol in POLICIES:
        for early in (0, 2):
            set_policy(*pol, early)
            F = to_dev(F0)
            F.lmxm(dA)
            n0 = launches(b"bits_pull_acc")
            F.union_lmxm([dA, dB])
            assert launches(b"bits_pull_acc") > n0, "the union hop did not accumulate through the pull"
            same(F, want2, f"union hop, hints/streams/hot_bytes {pol}, early_exit {early}")
