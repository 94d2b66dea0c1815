"""Full size: B200_expand_edges over RMAT-24 (edge factor 16, seed 1) split into 2 relationship types by a seeded edge hash, edge
ids in COO order, 10^5 multi-edge pairs per type (their ids in the host-resident me store), |dp| = |dm| = 10^6 per type, 1,024
sources including the 16 largest hubs.  OUT ALL, OUT FIRST and BOTH ALL must equal a vectorised numpy model over the same
layers: row pointers and every entry."""
import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200.grb import Matrix
from fullsize_util import need, rmat_both, defaults

pytestmark = pytest.mark.gpu
MULTI = np.uint64((1 << 64) - 1)


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def keys(r, c):
    return (r.astype(np.uint64) << np.uint64(32)) | c.astype(np.uint64)


def member(k, sorted_keys):
    if len(sorted_keys) == 0:
        return np.zeros(len(k), bool)
    q = np.minimum(np.searchsorted(sorted_keys, k), len(sorted_keys) - 1)
    return sorted_keys[q] == k


class Type:
    """one type's layers as numpy (m rows / cols / ids, dp, dm keys, me store) and on the device"""

    def __init__(self, n, rows, cols, ids, rng, id_next):
        nnz = len(rows)
        self.rows, self.cols, self.val = rows, cols, ids.copy()
        multi = rng.choice(nnz, 100_000, replace=False)
        self.val[multi] = MULTI
        mk = keys(rows[multi], cols[multi])
        extra = np.arange(id_next, id_next + len(multi), dtype=np.uint64)
        o = np.argsort(mk)
        self.me_key = np.repeat(mk[o], 2)
        self.me_id = np.stack([ids[multi][o], extra[o]], 1).reshape(-1)   # ids ascending inside a key (COO ids < extra ids)
        rest = np.setdiff1d(np.arange(nnz), multi)
        dmi = rng.choice(rest, 1_000_000, replace=False)
        self.dm = np.sort(keys(rows[dmi], cols[dmi]))
        dpr, dpc = rng.integers(0, n, 1_000_000).astype(np.uint64), rng.integers(0, n, 1_000_000).astype(np.uint64)
        dk, first = np.unique(keys(dpr, dpc), return_index=True)
        self.dp, self.dp_val = dk, np.arange(id_next + len(multi), id_next + len(multi) + len(dk), dtype=np.uint64)
        self.id_end = int(self.dp_val[-1]) + 1
        p = np.zeros(n + 1, np.uint64)
        np.cumsum(np.bincount(rows.astype(np.int64), minlength=n), out=p[1:])
        self.m_dev = Matrix.import_csr(n, n, p, cols.astype(np.uint32), self.val, "u64")
        pat = Matrix.import_csr(n, n, p, cols.astype(np.uint32), None, bool)
        self.mt_dev = pat.transpose()
        del pat
        r, c = self.dp >> np.uint64(32), self.dp & np.uint64(0xFFFFFFFF)
        self.dp_dev = Matrix(n, n, "u64")
        self.dp_dev.build(r, c, self.dp_val)
        self.mt_dp_dev = Matrix(n, n)
        self.mt_dp_dev.build(c, r)
        r, c = self.dm >> np.uint64(32), self.dm & np.uint64(0xFFFFFFFF)
        self.dm_dev = Matrix(n, n)
        self.dm_dev.build(r, c)
        self.mt_dm_dev = Matrix(n, n)
        self.mt_dm_dev.build(c, r)
        self.me_dev = Matrix(1 << 60, 1 << 60)
        self.me_dev.build(self.me_key, self.me_id)
        # the effective forward entries: m \ dm \ dp-shadowed, then dp (dp wins)
        k = keys(rows, cols)
        live = ~member(k, self.dm) & ~member(k, self.dp)
        self.eff_key = np.concatenate([k[live], self.dp])
        self.eff_val = np.concatenate([self.val[live], self.dp_val])

    def layers(self):
        return [self.m_dev, self.dp_dev, self.dm_dev, self.mt_dev, self.mt_dp_dev, self.mt_dm_dev, self.me_dev, None, None]

    def entries(self, sel):
        """(row, col, id) of the effective entries `sel` (a mask over eff_key), MULTI_EDGE expanded through me"""
        k, v = self.eff_key[sel], self.eff_val[sel]
        m = v == MULTI
        lo = np.searchsorted(self.me_key, k[m])
        hi = np.searchsorted(self.me_key, k[m], side="right")
        cnt = np.ones(len(k), np.int64)
        cnt[m] = hi - lo
        kk = np.repeat(k, cnt)
        ids = np.repeat(v, cnt)
        pos = np.repeat(np.cumsum(cnt) - cnt, cnt)
        slot = np.arange(len(kk)) - pos
        mrep = np.repeat(m, cnt)
        start = np.zeros(len(k), np.int64)
        start[m] = lo
        ids[mrep] = self.me_id[np.repeat(start, cnt)[mrep] + slot[mrep]]
        return kk >> np.uint64(32), kk & np.uint64(0xFFFFFFFF), ids


def model(types, src, dir, mode):
    """(p, node, edge, type, rev) over distinct sources"""
    order = np.argsort(src)
    S = src[order].astype(np.uint64)
    row_of = lambda x: order[np.searchsorted(S, x)]                 # the batch row of a (distinct) source
    parts = []
    for t, T in enumerate(types):
        r = T.eff_key >> np.uint64(32)
        c = T.eff_key & np.uint64(0xFFFFFFFF)
        fr, fc, fi = T.entries(member(r, S))
        parts.append((fr, fc, fi, np.full(len(fr), t), np.zeros(len(fr), np.uint8)))
        if dir == fb.DIR_BOTH:
            rr, rc, ri = T.entries(member(c, S) & (r != c))
            parts.append((rc, rr, ri, np.full(len(rr), t), np.ones(len(rr), np.uint8)))
    row = np.concatenate([row_of(x[0]) for x in parts]).astype(np.int64)
    node = np.concatenate([x[1] for x in parts]).astype(np.uint32)
    edge = np.concatenate([x[2] for x in parts])
    typ = np.concatenate([x[3] for x in parts]).astype(np.uint16)
    rev = np.concatenate([x[4] for x in parts])
    o = np.lexsort((edge, typ, node, rev, row))
    row, node, edge, typ, rev = row[o], node[o], edge[o], typ[o], rev[o]
    if mode == fb.EDGES_FIRST:
        keep = np.ones(len(row), bool)
        keep[1:] = (row[1:] != row[:-1]) | (rev[1:] != rev[:-1]) | (node[1:] != node[:-1])
        row, node, edge, typ, rev = row[keep], node[keep], edge[keep], typ[keep], rev[keep]
    p = np.zeros(len(src) + 1, np.uint64)
    np.cumsum(np.bincount(row, minlength=len(src)), out=p[1:])
    return p, node, edge, typ, rev


def test_expand_edges_rmat24_equals_the_numpy_model():
    need(40, 24)          # device: 2 typed bases with values and transposes, deltas; host: the graph, its split and the model
    scale, ntypes = 24, 2
    n = 1 << scale
    _, Ao = rmat_both(scale, 1)
    rng = np.random.default_rng(8)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(Ao.p))
    cols = Ao.j.astype(np.uint64)
    ids = np.arange(len(cols), dtype=np.uint64)                       # ids in COO order
    kind = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F))) >> np.uint64(63)
    types, id_next = [], len(cols)
    for t in range(ntypes):
        sel = np.nonzero(kind == t)[0]
        T = Type(n, rows[sel], cols[sel], ids[sel], rng, id_next)
        id_next = T.id_end
        types.append(T)
        del sel
    deg = np.diff(Ao.p.astype(np.int64))
    hubs = np.argsort(deg)[-16:]
    rest = rng.choice(np.setdiff1d(np.arange(n), hubs), 1024 - 16, replace=False)
    src = np.concatenate([hubs, rest]).astype(np.uint64)
    del rows, cols, ids, kind
    lays = [T.layers() for T in types]
    for dir, mode in ((fb.DIR_OUT, fb.EDGES_ALL), (fb.DIR_OUT, fb.EDGES_FIRST), (fb.DIR_BOTH, fb.EDGES_ALL)):
        got = fb.expand_edges(src, lays, dir, mode)
        want = model(types, src, dir, mode)
        what = f"dir={dir} mode={mode}"
        assert int(got[0][-1]) == int(want[0][-1]) > 0, f"{what}: {int(got[0][-1])} entries, the model has {int(want[0][-1])}"
        for name, x, y in zip(("p", "node", "edge", "type", "rev"), got, want):
            assert np.array_equal(x, y), f"{what}: {name} differs"
