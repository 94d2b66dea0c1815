"""Materialising a frontier bit-matrix as sorted CSR (bits.cu: bits_to_csr), checked against the CPU oracle on hand-built
frontiers.  The frontier is built as a CSR, turned into frontier form and multiplied by the identity, which keeps it in frontier
form (the diagonal column filter); waiting on the result then runs the count, scan and fill passes."""
import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200.grb import Matrix

pytestmark = pytest.mark.gpu

TILE = 1024      # vertices per fill tile


def frontier(rng, nrows, n):
    """Rows of every density: row 0 with every bit set, empty rows, sparse, half-dense and nearly full rows."""
    I, J = [], []
    for r in range(nrows):
        kind = (r + 1) % 7
        if kind == 0:
            continue                                    # empty row
        d = {1: 1.0 if r == 0 else 0.99, 2: 0.002, 3: 0.05, 4: 0.2, 5: 0.5, 6: 0.8}[kind]
        cols = np.nonzero(rng.random(n) < d)[0]
        I.append(np.full(len(cols), r, np.uint64))
        J.append(cols.astype(np.uint64))
    return np.concatenate(I), np.concatenate(J)


def segment_offsets_mod4(want, n):
    """output offset modulo 4 of every non-empty (row, tile) segment of the expected CSR"""
    seen = set()
    for r in range(want.nrows):
        cols = want.j[want.p[r]:want.p[r + 1]].astype(np.int64)
        if not len(cols):
            continue
        starts = np.searchsorted(cols, np.arange(0, n, TILE))
        nonempty = np.diff(np.append(starts, len(cols))) > 0
        seen |= set(((want.p[r] + starts[nonempty]) % 4).tolist())
    return seen


@pytest.mark.parametrize("nrows", [1, 64, 100, 128, 200, 256, 500, 512, 1000, 1024])   # W = 1, 1, 2, 2, 4, 4, 8, 8, 16, 16
@pytest.mark.parametrize("n", [700, 4096, 5000])                                          # below, on and off the tile size
def test_fill_matches_oracle(nrows, n):
    fb.init()
    fb.set_option("bits_mode", 1)
    try:
        rng = np.random.default_rng(nrows * 7919 + n)
        I, J = frontier(rng, nrows, n)
        want = orc.build_matrix(nrows, n, I, J)
        if nrows >= 64:
            assert segment_offsets_mod4(want, n) == {0, 1, 2, 3}
        ident = Matrix(n, n, bool)
        ident.build(np.arange(n, dtype=np.uint64), np.arange(n, dtype=np.uint64))
        F = Matrix(nrows, n, bool)
        F.build(I, J)
        F.lmxm(ident)
        assert fb.get_stat("last_path") == 5, "the product did not stay in frontier form"
        F.wait()
        p, j, _ = F.export_csr()
        assert np.array_equal(p, want.p), f"row pointers differ ({nrows} rows, n = {n})"
        assert np.array_equal(j, want.j), f"column indices differ ({nrows} rows, n = {n})"
        assert p[1] - p[0] == n, "the full row lost entries"
    finally:
        fb.set_option("bits_mode", -1)
