"""B200_adjacency_delta and the algo.pageRank / algo.WCC / algo.labelPropagation procedures over relationship operands with pending
writes.  The builder is compared, CSR for CSR and by digest, with a host model of the induced effective union; each procedure's device
route (one B200_adjacency_delta call) with the reference's route (a fresh matrix, or the compact walk over the tensors) and with the
oracle's PageRank / components / label propagation on the effective union; and the reference's flow-test expectations are replayed
from tests/golden/algo_flow_cases.json."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import falkordb_b200 as fb
import falkordb_b200.host_mirror as hm
import oracle as orc
from falkordb_b200._lib import lib
from falkordb_b200.grb import Matrix

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(autouse=True)
def _defaults():
    fb.init()
    yield
    fb.set_option("timing", 0)


def to_dev(n, pairs, dtype=bool):
    """an n x n matrix holding `pairs` (values 1.. for UINT64)"""
    pairs = sorted(set(pairs))
    c = orc.build_matrix(n, n, np.array([a for a, _ in pairs], np.int64), np.array([b for _, b in pairs], np.int64))
    x = np.arange(1, c.nnz + 1, dtype=np.uint64) if dtype == "u64" else None
    return Matrix.import_csr(n, n, c.p.astype(np.uint64), c.j, x, dtype)


def model(ops, n_out=None, keep=None, symmetric=False):
    """the induced effective union as an oracle CSR: U_t (m_t \\ dm_t) u dp_t (dp wins over dm), restricted to the vertices below
    n_out or to `keep`, renumbered by rank, with symmetric unioned with its transpose"""
    pairs = set()
    for m, dp, dm in ops:
        pairs |= (set(m) - set(dm or ())) | set(dp or ())
    if keep is None:
        rank = {v: v for v in range(n_out)}
        size = n_out
    else:
        rank = {int(v): k for k, v in enumerate(keep)}
        size = len(keep)
    out = {(rank[a], rank[b]) for a, b in pairs if a in rank and b in rank}
    if symmetric:
        out |= {(b, a) for a, b in out}
    out = sorted(out)
    return orc.build_matrix(size, size, np.array([a for a, _ in out], np.int64), np.array([b for _, b in out], np.int64))


def check_build(ops, dev_ops, n_out=None, keep=None, symmetric=False, what=""):
    A = fb.adjacency([o[0] for o in dev_ops], deltas=[(o[1], o[2]) for o in dev_ops], n=n_out, keep=keep, symmetric=symmetric)
    n = dev_ops[0][0].ncols()
    want = model(ops, n if n_out is None and keep is None else n_out, keep, symmetric)
    assert A.nrows() == A.ncols() == want.nrows, what
    p, j, _ = A.export_csr()
    assert np.array_equal(p, want.p) and np.array_equal(j, want.j), f"CSR differs {what}"
    assert np.array_equal(np.asarray(A.digest(), np.uint64), orc.digest(want)), f"digest differs {what}"
    return want


def random_operand(rng, A, ndel, nadd, overlap, outside, both):
    """host pair sets of one operand: m = A; dm = ndel entries of A + `outside` pairs not in A + `both` pairs also put into dp;
    dp = nadd new pairs + `overlap` entries of A + the `both` pairs"""
    n = A.nrows
    rows, cols, _ = A.tuples()
    m = list(zip(rows.tolist(), cols.tolist()))
    have = set(m)
    take = rng.choice(len(m), ndel + overlap + both, replace=False)
    fresh = lambda k: [t for t in zip(rng.integers(0, n, 4 * k + 8).tolist(), rng.integers(0, n, 4 * k + 8).tolist())
                       if t not in have and t[0] != t[1]][:k]
    dm = [m[i] for i in take[:ndel]] + fresh(outside)
    dp = fresh(nadd) + [m[i] for i in take[ndel:ndel + overlap]]
    shared = [m[i] for i in take[ndel + overlap:]] + fresh(both)
    return m, dp + shared, dm + shared


SCALE = 12
N = 1 << SCALE


@pytest.fixture(scope="module")
def world():
    """three RMAT operands with dirty deltas: operand 0 UINT64 (m and dp) with a BOOL dm, the others BOOL"""
    fb.init()
    rng = np.random.default_rng(9)
    ops, dev = [], []
    for t in range(3):
        A = orc.rmat_csr(SCALE, 6, 31 + t)
        m, dp, dm = random_operand(rng, A, ndel=800, nadd=400, overlap=30, outside=30, both=20)
        ops.append((m, dp, dm))
        dtype = "u64" if t == 0 else bool
        dev.append((to_dev(N, m, dtype), to_dev(N, dp, dtype), to_dev(N, dm)))
    keep = np.sort(rng.choice(N, N // 10, replace=False)).astype(np.uint64)
    return ops, dev, keep


@pytest.mark.parametrize("symmetric", [False, True])
@pytest.mark.parametrize("form", ["identity", "below_ncols", "keep"])
@pytest.mark.parametrize("nops", [1, 2, 3])
def test_builder_grid(world, nops, form, symmetric):
    ops, dev, keep = world
    kw = {"identity": {}, "below_ncols": {"n_out": N - 1000}, "keep": {"keep": keep}}[form]
    want = check_build(ops[:nops], dev[:nops], symmetric=symmetric, what=f"nops={nops} {form} symmetric={symmetric}", **kw)
    assert want.nnz > 100


def test_builder_clean_and_null_deltas(world):
    ops, dev, keep = world
    clean = [(m, None, None) for m, _, _ in ops]
    check_build(clean, [(d[0], None, None) for d in dev], what="NULL entries")
    A = fb.adjacency([d[0] for d in dev])                      # no deltas argument: NULL arrays
    p, j, _ = A.export_csr()
    want = model(clean, N)
    assert np.array_equal(p, want.p) and np.array_equal(j, want.j)
    check_build(clean[:1], [(dev[0][0], None, None)], keep=keep, symmetric=True, what="UINT64 base alone")


SMALL = 130     # three 64-id words, the last one partial


def small(ops, **kw):
    dev = [(to_dev(SMALL, m), to_dev(SMALL, dp) if dp else None, to_dev(SMALL, dm) if dm else None) for m, dp, dm in ops]
    return check_build(ops, dev, **kw)


def test_dp_wins_over_dm():
    for kw in ({}, {"keep": [0, 1, 5]}, {"symmetric": True}):
        want = small([([(0, 1), (1, 5)], [(0, 1)], [(0, 1), (1, 5)])], **kw)
        assert want.nnz >= 1


def test_entry_deleted_in_one_type_survives_in_another():
    want = small([([(0, 1), (1, 129)], None, [(0, 1)]), ([(0, 1)], None, None)])
    assert (0, 1) in want.tuple_set()
    want = small([([(0, 1)], None, [(0, 1)]), ([(2, 3)], [(0, 1)], None)], keep=[0, 1, 3])
    assert (0, 1) in want.tuple_set()


def test_dm_entry_outside_m_has_no_effect():
    want = small([([(0, 1), (64, 65)], None, [(3, 4), (64, 66), (127, 128)])], keep=[0, 1, 64, 65, 66])
    assert want.tuple_set() == {(0, 1), (2, 3)}


@pytest.mark.parametrize("keep", [[], [7], [63], [64], [63, 64], [0, 63, 64, 127, 128, 129], list(range(0, 130, 2))])
def test_kept_lists(keep):
    rng = np.random.default_rng(len(keep))
    pairs = lambda k: list({(int(a), int(b)) for a, b in zip(rng.integers(0, SMALL, k), rng.integers(0, SMALL, k))})
    ops = [(pairs(900), pairs(60), pairs(200)), (pairs(500), pairs(30), None)]
    for symmetric in (False, True):
        want = small(ops, keep=keep, symmetric=symmetric)
        assert want.nrows == len(keep)


def test_identity_form_sizes():
    ops = [([(0, 1), (5, 129), (129, 3), (100, 101)], [(128, 2)], [(100, 101)])]
    for n_out in (0, 1, 64, 100, 129, 130, 200):
        small(ops, n_out=n_out)
        small(ops, n_out=n_out, symmetric=True)


def test_reach_shares_the_builder(world):
    """the row-wise reach materialises its union through the same builder: bits_mode 0 gives the frontier path's result"""
    ops, dev, _ = world
    src = np.arange(0, 40, dtype=np.uint64)
    got = {}
    for mode in (0, -1):
        fb.set_option("bits_mode", mode)
        try:
            R, _ = fb.reach_batch(src, [d[0] for d in dev], max_hops=2, deltas=[(d[1], d[2]) for d in dev])
        finally:
            fb.set_option("bits_mode", -1)
        got[mode] = R.export_csr()[:2]
    assert np.array_equal(got[0][0], got[-1][0]) and np.array_equal(got[0][1], got[-1][1])


def test_timing_family():
    fb.set_option("timing", 1)
    fb.reset_stats()
    ops = [([(0, 1), (5, 129), (129, 3)], [(128, 2)], [(5, 129)])]
    small(ops, keep=[0, 1, 3, 129])
    ms, launches, nbytes = C.c_double(), C.c_uint64(), C.c_uint64()
    assert lib().B200_kernel_stats(b"adj_build", C.byref(ms), C.byref(launches), C.byref(nbytes)) == 0
    # one timed build per layer: m with its dm, then dp
    assert launches.value == 2 and nbytes.value > 0 and ms.value > 0


# ---- the procedures ----

HN = 3000
CAP = HN + 96           # the matrices' size (node_cap): ids run below HN, so the unfiltered matrix is cut to HN


def rel_err(a, b):
    if len(a) == 0:
        return 0.0
    return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300)))


@pytest.fixture(scope="module")
def graph():
    """two relationship types over HN nodes with multi-edges, pending inserts and deletes; the adjacency VersionedMatrix holding
    their effective union; three label matrices (diagonals, one with a pending removal) and a set of deleted nodes that hold no
    label and no edge"""
    fb.init()
    rng = np.random.default_rng(17)
    nxt = [0]

    def ids(k):
        nxt[0] += k
        return np.arange(nxt[0] - k, nxt[0], dtype=np.uint64)

    deleted = sorted(rng.choice(HN, 40, replace=False).tolist())
    dead = set(deleted)
    live = np.array([v for v in range(HN) if v not in dead])
    types, held = [], []
    for t in range(2):
        s, d = rng.choice(live, 4200), rng.choice(live, 4200)
        s, d = np.concatenate([s, s[:200]]), np.concatenate([d, d[:200]])          # multi-edges
        e = ids(len(s))
        T = hm.Tensor(CAP, s, d, e)
        rel = {int(x): (int(a), int(b)) for x, a, b in zip(e, s, d)}
        ns, nd = rng.choice(live, 500), rng.choice(live, 500)
        ne = ids(500)
        T.add(ns, nd, ne)                                                          # pending inserts
        rel.update({int(x): (int(a), int(b)) for x, a, b in zip(ne, ns, nd)})
        gone = rng.choice(sorted(rel), 700, replace=False)                         # pending deletes
        T.remove(gone, [rel[int(x)][0] for x in gone], [rel[int(x)][1] for x in gone])
        for x in gone:
            del rel[int(x)]
        types.append(T)
        held.append(set(rel.values()))
    adj = hm.VersionedMatrix(CAP)
    for a, b in sorted(held[0] | held[1]):
        adj.set(a, b)
    labels, members = [], []
    for frac in (0.01, 0.1, 0.5):
        vs = sorted(rng.choice(live, max(2, int(frac * len(live))), replace=False).tolist())
        L = hm.VersionedMatrix(CAP)
        for v in vs:
            L.set(v, v)
        if frac == 0.5:
            L.remove(vs[0], vs[0])                                                 # a pending removal from the label
            vs = vs[1:]
        labels.append(L)
        members.append(vs)
    everyone = hm.VersionedMatrix(CAP)
    for v in live:
        everyone.set(int(v), int(v))
    return dict(adj=adj, types=types, held=held, labels=labels, members=members, everyone=everyone, deleted=deleted,
                node_count=HN - len(deleted))


def expected(g, proc, named, label_ids, max_iterations=10):
    """(nodes, values) of the procedure on the oracle: label_ids None = unfiltered"""
    n_out = g["node_count"] + len(g["deleted"])
    pairs = set().union(*[g["held"][k] for k in (named if named else (0, 1))])
    ops = [(sorted(pairs), None, None)]
    keep = None if label_ids is None else sorted(set(label_ids))
    A = model(ops, n_out=n_out if keep is None else None, keep=keep, symmetric=proc != "pagerank")
    if proc == "pagerank":
        vals, _ = orc.pagerank(A, float(np.float32(0.85)), float(np.float32(1e-4)), 100)
    elif proc == "wcc":
        vals = orc.wcc(A)
    else:
        vals, _ = orc.cdlp(A, max_iterations)
    ids = np.arange(A.nrows) if keep is None else np.array(keep, np.int64)
    dead = set(g["deleted"])
    alive = np.array([int(v) not in dead for v in ids], bool)
    return ids[alive].astype(np.uint64), vals[alive] if len(vals) else vals


def run_both(g, proc, named, labels, **kw):
    fn = {"pagerank": hm.algo_pagerank, "wcc": hm.algo_wcc, "cdlp": hm.algo_cdlp}[proc]
    args = (g["adj"], g["types"], [g["types"][k] if k is not None else None for k in named], labels, g["node_count"], g["deleted"])
    got = fn(*args, route=hm.ALGO_DEVICE, **kw)
    want = fn(*args, route=hm.ALGO_BY_EXTRACT, **kw)
    assert np.array_equal(got[0], want[0]), f"{proc}: node columns differ"
    assert np.array_equal(got[1], want[1]), f"{proc}: value columns differ"      # pageRank bit for bit: same kernel, same CSR
    return got


@pytest.mark.parametrize("named", [(), (0,), (1,), (0, 1)])
@pytest.mark.parametrize("label", [None, 0, 1, 2, "all"])
@pytest.mark.parametrize("proc", ["pagerank", "wcc", "cdlp"])
def test_procedures_match_the_reference_route_and_the_oracle(graph, proc, label, named):
    g = graph
    if label is None:
        labels, ids = [], None
    elif label == "all":                          # pageRank: a label covering every node runs unfiltered
        dead = set(g["deleted"])
        labels, ids = [g["everyone"]], None if proc == "pagerank" else [v for v in range(HN) if v not in dead]
    else:
        labels, ids = [g["labels"][label]], g["members"][label]
    nodes, vals = run_both(g, proc, named, labels)
    wn, wv = expected(g, proc, named, ids)
    assert np.array_equal(nodes, wn)
    assert not set(nodes.tolist()) & set(g["deleted"])
    if proc == "pagerank":
        assert rel_err(vals, wv) < 1e-12, f"scores rel err {rel_err(vals, wv)}"
    else:
        assert np.array_equal(vals, wv.astype(np.int64))


@pytest.mark.parametrize("proc", ["wcc", "cdlp"])
def test_node_label_unions(graph, proc):
    g = graph
    nodes, vals = run_both(g, proc, (1,), [g["labels"][0], g["labels"][2]])
    wn, wv = expected(g, proc, (1,), g["members"][0] + g["members"][2])
    assert np.array_equal(nodes, wn) and np.array_equal(vals, wv.astype(np.int64))


def test_cdlp_max_iterations(graph):
    g = graph
    for it in (1, 3):
        nodes, vals = run_both(g, "cdlp", (), [], max_iterations=it)
        wn, wv = expected(g, "cdlp", (), None, it)
        assert np.array_equal(nodes, wn) and np.array_equal(vals, wv.astype(np.int64))


def test_missing_names_and_empty_results(graph):
    g = graph
    # a type the graph does not have contributes nothing
    for proc in ("pagerank", "wcc", "cdlp"):
        nodes, vals = run_both(g, proc, (None,), [])
        assert len(nodes) == g["node_count"]
        nodes2, _ = run_both(g, proc, (None, 1), [g["labels"][1]])
        wn, _ = expected(g, proc, (1,), g["members"][1])
        assert np.array_equal(nodes2, wn)
    # WCC / CDLP: an empty node set returns nothing; pageRank runs on a 0 x 0 matrix
    for proc in ("pagerank", "wcc", "cdlp"):
        nodes, vals = run_both(g, proc, (), [None])
        assert len(nodes) == 0 and len(vals) == 0
    # no live node: nothing
    fn = hm.algo_wcc
    for route in (hm.ALGO_DEVICE, hm.ALGO_BY_EXTRACT):
        nodes, vals = fn(g["adj"], g["types"], [], [], 0, [], route=route)
        assert len(nodes) == 0


def test_reference_flow_expectations():
    cases = json.load(open(os.path.join(HERE, "golden", "algo_flow_cases.json")))
    for case in cases["cases"]:
        gd = cases["graphs"][case["graph"]]
        names = [nm for nm, _ in gd["nodes"]]
        n = len(names)
        type_names = sorted({t for _, _, t in gd["edges"]})
        tensors = {}
        for k, tn in enumerate(type_names):
            es = [(a, b) for a, b, t in gd["edges"] if t == tn]
            tensors[tn] = hm.Tensor(n, [a for a, _ in es], [b for _, b in es], np.arange(len(es)) + 1000 * k)
        adj = hm.VersionedMatrix(n)
        for a, b, _ in gd["edges"]:
            adj.set(a, b)
        label_mats = {}
        for v, (_, ls) in enumerate(gd["nodes"]):
            for lab in ls:
                label_mats.setdefault(lab, hm.VersionedMatrix(n)).set(v, v)
        named = [tensors.get(t) for t in (case["relationshipTypes"] or [])]
        labels = [label_mats.get(lab) for lab in (case["nodeLabels"] or [])]
        fn = hm.algo_wcc if case["proc"] == "wcc" else hm.algo_cdlp
        out = []
        for route in (hm.ALGO_DEVICE, hm.ALGO_BY_EXTRACT):
            nodes, ids = fn(adj, [tensors[t] for t in type_names], named, labels, n, [], route=route)
            out.append((nodes, ids))
        assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1]), case
        nodes, ids = out[0]
        comp = {}
        for v, c in zip(nodes.tolist(), ids.tolist()):
            comp.setdefault(c, []).append(names[v])
        if "components" in case:
            got = sorted(sorted(c) for c in comp.values())
            assert got == sorted(sorted(c) for c in case["components"]), (case, got)
        else:
            of = {names[v]: c for v, c in zip(nodes.tolist(), ids.tolist())}
            heads = []
            for grp in case["groups"]:
                assert len({of[x] for x in grp}) == 1, (case, grp)
                heads.append(of[grp[0]])
            assert len(set(heads)) == len(heads), case
            if "nodes" in case:
                assert sorted(names[v] for v in nodes.tolist()) == sorted(case["nodes"]), case
