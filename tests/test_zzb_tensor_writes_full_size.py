"""Full size: relationship writes through the reference route (Tensor::set_all_from_slices / remove_all, read phase on the host)
and the device route (set_all_from_slices_dev / remove_all_dev, B200_Tensor_insert_plan / _remove_plan) on RMAT-24 (edge factor 16,
seed 1) split into 3 relationship types by a seeded edge hash, 1 % of pairs with a second edge, each type loaded twice by
Tensor::bulk_load.  Per type: 10^6 inserts (3/4 random pairs, 1/4 loaded pairs: promotions), then 10^6 deletes (half the ids on
multi-edge pairs).  The twins must agree: digests of m and mt's base, every entry of the other seven layers (me included), the
six Delta counters, edge_count and the emptied pairs."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from fullsize_util import need, rmat_both, defaults

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _defaults():
    yield from defaults()


def state(t):
    out = []
    for k, h in enumerate(t.layers()):
        if k in (0, 3):
            d = np.zeros(3, np.uint64)
            fb.check(fb.lib().B200_Matrix_digest(C.c_void_p(h), d.ctypes.data))
            out.append(("digest", k, d))
        else:
            out.extend(("tuples", k, x) for x in hm._tuples(h, k < 2) if x is not None)
    out.append(("counters", -1, t.counts()))
    out.append(("edge_count", -1, np.array([t.edge_count()], np.uint64)))
    return out


def assert_same(a, b, what):
    for (kind, k, x), (_, _, y) in zip(state(a), state(b)):
        assert np.array_equal(x, y), f"{what}: {kind} of layer {k} differs"


def test_writes_rmat24_three_types_equal_on_both_routes():
    need(24, 40)          # device: 6 bases with values and transposes; host: the graph, its split, the reference route's downloads
    scale, T, batch = 24, 3, 1_000_000
    n = 1 << scale
    _, Ao = rmat_both(scale, 1)
    rng = np.random.default_rng(12)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(Ao.p))
    cols = Ao.j.astype(np.uint64)
    ids = np.arange(len(cols), dtype=np.uint64)
    extra = rng.choice(len(cols), len(cols) // 100, replace=False)
    multi = np.zeros(len(cols) + len(extra), bool)
    multi[extra] = True
    multi[len(cols):] = True
    rows, cols = np.concatenate([rows, rows[extra]]), np.concatenate([cols, cols[extra]])
    ids = np.concatenate([ids, np.arange(len(ids), len(ids) + len(extra), dtype=np.uint64)])
    kind = (((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F))) >> np.uint64(61)) % np.uint64(T)
    next_id = len(ids)
    for t in range(T):
        sel = np.nonzero(kind == t)[0]
        ref, dev = hm.Tensor(n, rows[sel], cols[sel], ids[sel]), hm.Tensor(n, rows[sel], cols[sel], ids[sel])
        q = batch - batch // 4
        old = rng.choice(sel, batch // 4)
        ns = np.concatenate([rng.integers(0, n, q).astype(np.uint64), rows[old]])
        nd = np.concatenate([rng.integers(0, n, q).astype(np.uint64), cols[old]])
        nid = np.arange(next_id, next_id + batch, dtype=np.uint64)
        next_id += batch
        ref.add(ns, nd, nid, route=hm.WRITE_REFERENCE)
        dev.add(ns, nd, nid, route=hm.WRITE_DEVICE)
        assert_same(ref, dev, f"type {t} after the inserts")
        ms, ss = sel[multi[sel]], sel[~multi[sel]]
        g = np.concatenate([rng.choice(ms, batch // 2, replace=False), rng.choice(ss, batch - batch // 2, replace=False)])
        e1 = ref.remove(ids[g], rows[g], cols[g], route=hm.WRITE_REFERENCE)
        e2 = dev.remove(ids[g], rows[g], cols[g], route=hm.WRITE_DEVICE)
        assert len(e2) > 0 and set(map(tuple, e1.tolist())) == set(map(tuple, e2.tolist())), f"type {t}: emptied pairs differ"
        assert_same(ref, dev, f"type {t} after the deletes")
        del ref, dev
