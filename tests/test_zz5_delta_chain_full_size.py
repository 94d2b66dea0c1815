"""Full size: a dirty 3-hop chain on RMAT-24 (edge factor 16, seed 1) from 512 sources, every hop's operand (m, dp, dm) with
|dp| = |dm| = 10^6.  The fused chain (B200_Matrix_delta_lmxm per hop) and the reference's composition (three GrB_mxm plus an
eWiseAdd per hop, Matrix.delta_lmxm) must give identical digests, nvals and flops."""
import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200.grb import Matrix
from fullsize_util import need, rmat_both, defaults

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def test_dirty_three_hop_chain_rmat24_fused_equals_composition():
    need(40, 8)           # device: graph + transpose + 3 frontiers of 1.07 GB + the 6.8 GB digest CSR; host: the exported graph
    scale, nsrc, ndelta = 24, 512, 1_000_000
    n = 1 << scale
    A, Ao = rmat_both(scale, 1)
    A.prepare(True)
    rng = np.random.default_rng(1)
    pick = np.sort(rng.choice(Ao.nnz, size=ndelta, replace=False))
    dm = Matrix(n, n, bool)
    dm.build((np.searchsorted(Ao.p, pick, side="right") - 1).astype(np.uint64), Ao.j[pick].astype(np.uint64))
    dp = Matrix(n, n, bool)
    dp.build(rng.integers(0, n, ndelta).astype(np.uint64), rng.integers(0, n, ndelta).astype(np.uint64))
    src = rng.choice(np.nonzero(np.diff(Ao.p))[0], nsrc, replace=False)

    def chain(fused):
        F = Matrix(nsrc, n, bool)
        F.build(np.arange(nsrc), src)
        fb.reset_stats()
        for _ in range(3):
            (F.delta_lmxm_fused if fused else F.delta_lmxm)(A, dp, dm)
        return F, fb.get_stat("total_flops")

    G, flops_c = chain(False)
    dg_c, nv_c = G.digest(), G.nvals()
    del G
    F, flops_f = chain(True)
    assert F.nvals() == nv_c and nv_c > 0
    assert np.array_equal(F.digest(), dg_c), "fused and composed dirty chains differ"
    assert flops_f == flops_c
