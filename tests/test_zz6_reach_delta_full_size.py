"""Full size: reachability over RMAT-24 (edge factor 16, seed 1) with pending writes, 512 sources, max_hops = 3, |dp| = |dm| = 10^6.
B200_reach_batch_delta must give what B200_reach_batch gives on the materialised operand (m \\ dm) u dp -- digest, nvals and
levels -- with one operand, and with two (m and its transpose, each with its own deltas)."""
import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200.grb import Descriptor, Matrix
from fullsize_util import need, rmat_both, defaults

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def materialise(n, m, dp, dm):
    """(m \\ dm) u dp through the library's own set operations"""
    E = Matrix(n, n, bool)
    E.element_wise_add(dm, m, m, Descriptor.RC)          # E<!dm, replace> = m
    E.element_wise_add(None, E, dp)
    return E


def test_dirty_reach_rmat24_equals_reach_over_the_materialised_operand():
    need(40, 8)           # device: graph, transpose, the materialised operands with their mirrors; host: the exported graph
    scale, nsrc, ndelta, hops = 24, 512, 1_000_000, 3
    n = 1 << scale
    A, Ao = rmat_both(scale, 1)
    A.prepare(True)
    rng = np.random.default_rng(2)
    pick = np.sort(rng.choice(Ao.nnz, size=ndelta, replace=False))
    rows = (np.searchsorted(Ao.p, pick, side="right") - 1).astype(np.uint64)
    cols = Ao.j[pick].astype(np.uint64)
    prs, pcs = rng.integers(0, n, ndelta).astype(np.uint64), rng.integers(0, n, ndelta).astype(np.uint64)
    dm, dp, dmT, dpT = (Matrix(n, n, bool) for _ in range(4))
    dm.build(rows, cols)
    dp.build(prs, pcs)
    dmT.build(cols, rows)
    dpT.build(pcs, prs)
    At = A.transpose().prepare(True)
    src = rng.choice(np.nonzero(np.diff(Ao.p))[0], nsrc, replace=False)

    E = materialise(n, A, dp, dm)
    R0, l0 = fb.reach_batch(src, E, hops)
    R1, l1 = fb.reach_batch(src, [A], hops, deltas=[(dp, dm)])
    assert l1 == l0 == hops and R1.nvals() == R0.nvals() > 0
    assert np.array_equal(R1.digest(), R0.digest()), "one operand: dirty reach differs from the reach over (m \\ dm) u dp"
    del R0, R1

    U = Matrix(n, n, bool)
    U.element_wise_add(None, E, materialise(n, At, dpT, dmT))
    del E
    R0, l0 = fb.reach_batch(src, U, hops)
    R1, l1 = fb.reach_batch(src, [A, At], hops, deltas=[(dp, dm), (dpT, dmT)])
    assert l1 == l0 and R1.nvals() == R0.nvals() > 0
    assert np.array_equal(R1.digest(), R0.digest()), "two operands: dirty reach differs from the reach over the union"
