"""Full size: algo.BFS over RMAT-24 (edge factor 16, seed 1) split into 3 relationship types by an edge hash, each with
|dp| = |dm| = 10^5 pending, from 4 sources.  B200_bfs_delta must give the levels and parents of B200_bfs_ex on the prepared
materialised union, and of the oracle for one source."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
import oracle as orc
from falkordb_b200._lib import lib, BfsInfo
from falkordb_b200.grb import Descriptor, Matrix
from fullsize_util import need, rmat_both, defaults

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def test_dirty_bfs_rmat24_three_types_equals_bfs_over_the_materialised_union():
    need(30, 16)          # device: the types with their mirrors, the union with its mirror; host: the exported graph and its split
    scale, ntypes, ndelta, nsrc = 24, 3, 100_000, 4
    n = 1 << scale
    _, Ao = rmat_both(scale, 1)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(Ao.p))
    cols = Ao.j.astype(np.uint64)
    kind = (((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F))) >> np.uint64(61)) % np.uint64(ntypes)
    rng = np.random.default_rng(4)
    ops = []
    for t in range(ntypes):
        sel = np.nonzero(kind == t)[0]
        pt = np.zeros(n + 1, np.uint64)
        np.cumsum(np.bincount(rows[sel].astype(np.int64), minlength=n), out=pt[1:])
        m = Matrix.import_csr(n, n, pt, Ao.j[sel], None, bool)
        pick = rng.choice(len(sel), ndelta, replace=False)
        dm, dp = Matrix(n, n, bool), Matrix(n, n, bool)
        dm.build(rows[sel][pick], cols[sel][pick])
        dp.build(rng.integers(0, n, ndelta).astype(np.uint64), rng.integers(0, n, ndelta).astype(np.uint64))
        ops.append((m, dp, dm))
    del rows, cols, kind
    U = Matrix(n, n, bool)
    for m, dp, dm in ops:                       # U |= (m \ dm) u dp, through the library's own set operations
        E = Matrix(n, n, bool)
        E.element_wise_add(dm, m, m, Descriptor.RC)
        E.element_wise_add(None, E, dp)
        U.element_wise_add(None, U, E)
        del E
    U.prepare(True)
    src = rng.choice(np.nonzero(np.diff(Ao.p))[0], nsrc, replace=False)
    for k, s in enumerate(src):
        info = BfsInfo()
        lv, pr, _ = fb.bfs([o[0] for o in ops], int(s), deltas=[(o[1], o[2]) for o in ops], info=info)
        el, ep = np.empty(n, np.int64), np.empty(n, np.int64)
        fb.check(lib().B200_bfs_ex(U.h, int(s), -1, -1, el.ctypes.data, ep.ctypes.data, 0, None))
        assert (lv >= 0).sum() > n // 4 and info.bu_levels > 0
        assert np.array_equal(lv, el), f"source {s}: levels differ from the BFS over the materialised union"
        assert np.array_equal(pr, ep), f"source {s}: parents differ from the BFS over the materialised union"
        if k == 0:
            p, j, _ = U.export_csr()
            wl, wp = orc.bfs(orc.CSR(n, n, p, j), int(s))
            del p, j
            assert np.array_equal(lv, wl) and np.array_equal(pr, wp), f"source {s}: differs from the oracle"
