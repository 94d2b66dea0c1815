"""Full size: a 3-hop chain of union hops over RMAT-24 (edge factor 16, seed 1) split into 3 relationship types by a seeded edge
hash, |dp| = |dm| = 10^6 per type, 512 sources.  The union hops (B200_Matrix_union_lmxm per hop, and B200_traverse_batch_union)
must give what the reference's route gives -- union_by_extract, then a hop by the fresh matrix: digest, nvals and the bitmap --
and report sum_t flops(F*m_t) + flops(F*dp_t) per hop."""
import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200.grb import Descriptor, Matrix
from fullsize_util import need, rmat_both, defaults

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def union_by_extract(n, ops):
    """graph.rs:2520-2550: extract(T_1), then set_pattern(<!dm_t> m_t) and set_pattern(dp_t) per further type"""
    U = Matrix(n, n, bool)
    m, dp, dm = ops[0]
    U.set_pattern(None, m)
    U.remove_all(dm)
    U.set_pattern(None, dp)
    for m, dp, dm in ops[1:]:
        U.set_pattern(dm, m, Descriptor.C)
        U.set_pattern(None, dp)
    U.wait()
    return U


def last_flops(out, F, B):
    out.mxm(F, B)
    return fb.get_stat("last_flops")


def test_union_chain_rmat24_equals_the_extract_route():
    need(48, 12)          # device: graph, 3 types with mirrors, the union with its mirror, frontiers; host: graph + 2 bitmaps
    scale, nsrc, ndelta, hops, ntypes = 24, 512, 1_000_000, 3, 3
    n = 1 << scale
    _, Ao = rmat_both(scale, 1)
    rng = np.random.default_rng(4)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(Ao.p))
    cols = Ao.j.astype(np.uint64)
    kind = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F)) ^ np.uint64(7)) >> np.uint64(61)
    kind = (kind % np.uint64(ntypes)).astype(np.int8)
    ops = []
    for t in range(ntypes):
        sel = np.nonzero(kind == t)[0]
        p = np.zeros(n + 1, np.uint64)
        np.cumsum(np.bincount(rows[sel].astype(np.int64), minlength=n), out=p[1:])
        m = Matrix.import_csr(n, n, p, Ao.j[sel], None, bool).prepare(True)
        pick = rng.choice(len(sel), size=ndelta, replace=False)
        dm, dp = Matrix(n, n, bool), Matrix(n, n, bool)
        dm.build(rows[sel][pick], cols[sel][pick])
        dp.build(rng.integers(0, n, ndelta).astype(np.uint64), rng.integers(0, n, ndelta).astype(np.uint64))
        ops.append((m, dp, dm))
        del sel, pick
    del rows, cols, kind
    U = union_by_extract(n, ops).prepare(True)
    src = rng.choice(np.nonzero(np.diff(Ao.p))[0], nsrc, replace=False)

    F0, F1 = Matrix(nsrc, n, bool), Matrix(nsrc, n, bool)
    for F in (F0, F1):
        F.build(np.arange(nsrc), src)
    want_fl = got_fl = 0
    for h in range(hops):
        T = Matrix(nsrc, n, bool)
        want_fl += sum(last_flops(T, F0, m) + last_flops(T, F0, dp) for m, dp, _ in ops)
        del T
        F0.mxm(F0, U)
        F1.union_lmxm([o[0] for o in ops], [(o[1], o[2]) for o in ops])
        got_fl += fb.get_stat("last_flops")
        assert F1.nvals() == F0.nvals() > 0, f"hop {h + 1}: nvals"
        assert np.array_equal(F1.digest(), F0.digest()), f"hop {h + 1}: the union hop differs from the extract route"
    assert got_fl == want_fl, "union hop flops are not sum_t flops(F*m_t) + flops(F*dp_t)"
    del F0, F1

    wpr = n // 64
    b0, b1 = np.zeros((nsrc, wpr), np.uint64), np.zeros((nsrc, wpr), np.uint64)
    fb.traverse_batch(src, [U] * hops, fb.OUT_BITMAP, out_bitmap=b0)
    fl, _, _ = fb.traverse_batch(src, [[o[0] for o in ops]] * hops, fb.OUT_BITMAP, out_bitmap=b1,
                                 deltas=[[(o[1], o[2]) for o in ops]] * hops)
    assert fl == want_fl, "B200_traverse_batch_union flops"
    assert np.array_equal(b0, b1), "B200_traverse_batch_union differs from B200_traverse_batch over the extracted union"
