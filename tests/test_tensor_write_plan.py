"""B200_Tensor_insert_plan / B200_Tensor_remove_plan and the host mirror's device write route (Tensor::set_all_from_slices_dev /
remove_all_dev, VersionedMatrix::set_all_dev) on the GPU:
- the plan arrays against a restatement of the two tables in include/b200grb.h over random raw layers;
- the transcribed tensor.rs tests through both write routes;
- a seeded model check: twin tensors, one written through each route, equal after every step (nine layers tuple for tuple, the six
  Delta counters, edge_count, emptied pairs);
- a bulk-loaded base is not downloaded by device-route writes (d2h_bytes), while the reference route downloads it;
- set_all_dev equals set_all, with dm empty and not."""
import ctypes as C

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from falkordb_b200.grb import Matrix, PLAN_COMMITTED, PLAN_CANCEL, PLAN_MT_BASE, PLAN_EMPTIED, PLAN_DEMOTED, PLAN_M_HAS, PLAN_M_EQ

pytestmark = pytest.mark.gpu
MULTI = (1 << 64) - 1


@pytest.fixture(autouse=True)
def _init():
    fb.init()
    yield


def key(s, d):
    return (int(s) << 32) | int(d)


# ---- plan arrays against the tables ----
class Layers:
    """random raw layers of one type (dicts / sets) and the same as library matrices"""

    def __init__(self, rng, n=32):
        self.n = n
        pairs = lambda k: {(int(a), int(b)) for a, b in rng.integers(0, n, (k, 2))}
        self.m = {p: (MULTI if rng.random() < 0.25 else int(rng.integers(0, 1000))) for p in pairs(160)}
        self.dp = {p: (MULTI if rng.random() < 0.25 else int(rng.integers(0, 1000))) for p in pairs(50)}
        self.dm = {p for p in self.m if p not in self.dp and rng.random() < 0.2} | {p for p in pairs(6) if p not in self.dp}
        self.mt = {(d, s) for (s, d) in self.m if rng.random() < 0.8} | {(d, s) for (s, d) in pairs(10)}
        multi = [key(*p) for p, v in list(self.m.items()) + list(self.dp.items()) if v == MULTI]
        self.me = {(k, int(i)) for k in multi for i in rng.choice(3000, int(rng.integers(2, 6)), replace=False)}
        mel = sorted(self.me)
        self.me_dm = {mel[i] for i in rng.choice(len(mel), len(mel) // 5, replace=False)}
        self.me_dp = {(k, int(i)) for k in multi for i in rng.choice(3000, int(rng.integers(0, 3)), replace=False)} - self.me
        self.dev = {"m": self._u64(self.m), "dp": self._u64(self.dp), "dm": self._bool(self.dm, n), "mt": self._bool(self.mt, n),
                    "mt_dp": Matrix(n, n), "mt_dm": Matrix(n, n), "me": self._bool(self.me, 1 << 60),
                    "me_dp": self._bool(self.me_dp, 1 << 60), "me_dm": self._bool(self.me_dm, 1 << 60)}

    def _u64(self, d):
        M = Matrix(self.n, self.n, "u64")
        if d:
            k = sorted(d)
            M.build([a for a, _ in k], [b for _, b in k], [d[p] for p in k])
        return M

    @staticmethod
    def _bool(s, dim):
        M = Matrix(dim, dim)
        if s:
            k = sorted(s)
            M.build([a for a, _ in k], [b for _, b in k])
        return M

    def merged(self, k):
        return sorted({i for kk, i in self.me if kk == k and (kk, i) not in self.me_dm} | {i for kk, i in self.me_dp if kk == k})

    def eff(self, p):
        if p in self.dp:
            return self.dp[p]
        if p in self.dm:
            return None
        return self.m.get(p)


def model_insert(L, srcs, dsts, ids):
    runs = {}
    for s, d, i in zip(srcs, dsts, ids):
        runs.setdefault((int(s), int(d)), []).append(int(i))
    rec, me = [], []
    for p in sorted(runs):
        its, (s, d), k = runs[p], p, key(*p)
        cur = L.dp[p] if p in L.dp else (None if p in L.dm else L.m.get(p))
        if cur == MULTI:
            ent, inl = its, None
        elif cur is not None:
            ent, inl, committed = [cur] + its, MULTI, p in L.dp and p in L.m
        else:
            ent, inl, committed = (its if len(its) > 1 else []), (MULTI if len(its) > 1 else its[0]), p in L.dm and p in L.m
        if inl is not None:
            f = (PLAN_COMMITTED if committed else 0) | (PLAN_CANCEL if committed and L.m[p] == inl else 0)
            f |= PLAN_MT_BASE if (d, s) in L.mt else 0
            rec.append((s, d, inl, f))
        me += [(k, i, (k, i) in L.me) for i in ent]
    return rec, me


def model_remove(L, ids, srcs, dsts):
    runs = {}
    for i, s, d in zip(ids, srcs, dsts):
        runs.setdefault((int(s), int(d)), set()).add(int(i))
    rec, me = [], []
    for p in sorted(runs):
        R, (s, d), k = runs[p], p, key(*p)
        v = L.eff(p)
        f, val, ent = 0, v, []
        if v is None:
            continue
        if v != MULTI:
            f = PLAN_EMPTIED if v in R else 0
        else:
            lst = L.merged(k)
            H = [i for i in lst if i in R]
            rem = [i for i in lst if i not in R]
            if not H:
                continue
            if len(rem) >= 2 or len(lst) < 2:                       # a one-id list (a live id added twice): the ids named go
                ent = H
            else:
                ent = lst
                f = PLAN_DEMOTED if rem else PLAN_EMPTIED
                val = rem[0] if rem else v
        if f:
            f |= PLAN_M_HAS if p in L.m else 0
            f |= PLAN_M_EQ if (f & PLAN_DEMOTED) and L.m.get(p) == val else 0
            f |= PLAN_MT_BASE if (d, s) in L.mt else 0
            rec.append((s, d, val, f))
        me += [(k, i, (k, i) in L.me) for i in ent]
    return rec, me


def as_lists(p):
    rec = list(zip(*(p[x].tolist() for x in ("src", "dst", "val", "flags"))))
    me = list(zip(p["me_key"].tolist(), p["me_id"].tolist(), p["me_base"].tolist()))
    return rec, me


@pytest.mark.parametrize("seed", range(4))
def test_plan_arrays_match_the_tables(seed):
    rng = np.random.default_rng(seed)
    L = Layers(rng)
    known = sorted(set(L.m) | set(L.dp) | L.dm)
    seen = 0
    for trial in range(6):
        k = int(rng.integers(1, 60))
        pick = [known[i] for i in rng.integers(0, len(known), k)] + [tuple(map(int, x)) for x in rng.integers(0, L.n, (k // 3, 2))]
        pick += pick[: k // 4]                                           # in-batch duplicates
        order = rng.permutation(len(pick))
        srcs = [pick[i][0] for i in order]
        dsts = [pick[i][1] for i in order]
        ids = [int(x) for x in rng.integers(0, 1000, len(pick))]
        ids[0] = 0
        want = model_insert(L, srcs, dsts, ids)
        got = as_lists(fb.insert_plan(L.dev, srcs, dsts, ids))
        assert got == want, f"insert plan, seed {seed} trial {trial}"
        # removes: every id of some multi pairs (empty), all but one (demote), some (stay), singles, stale and repeated ids
        rel = []
        for p in known:
            v, r = L.eff(p), rng.random()
            if v is None:
                if r < 0.1:
                    rel.append((5, *p))
            elif v != MULTI:
                if r < 0.5:
                    rel.append((v if r < 0.35 else v + 1, *p))
            else:
                lst = L.merged(key(*p))
                take = lst if r < 0.3 else lst[1:] if r < 0.6 else lst[: max(0, len(lst) - 2)] if r < 0.8 else []
                rel += [(i, *p) for i in take] + [(9999, *p)] * (r > 0.9)
        rel += rel[: len(rel) // 5]
        rel = [rel[i] for i in rng.permutation(len(rel))]
        ids_r, s_r, d_r = [x[0] for x in rel], [x[1] for x in rel], [x[2] for x in rel]
        want = model_remove(L, ids_r, s_r, d_r)
        got = as_lists(fb.remove_plan(L.dev, ids_r, s_r, d_r))
        assert got == want, f"remove plan, seed {seed} trial {trial}"
        for *_, f in want[0]:
            seen |= f
    assert seen & PLAN_DEMOTED and seen & PLAN_EMPTIED and seen & PLAN_M_HAS


# ---- the transcribed tensor.rs tests through both routes ----
WRITE_TESTS = ["multi_pairs_after_within_batch_duplicates", "multi_pairs_matches_the_sentinel_count",
               "bulk_remove_and_extract_edge_id_zero", "deleting_everything_folds_the_tombstones_away",
               "batch_demote_leaves_every_survivor_inline", "batch_can_demote_and_then_empty_the_same_pair",
               "demoting_to_the_committed_value_cancels_to_clean"]


@pytest.mark.parametrize("route", [hm.WRITE_REFERENCE, hm.WRITE_DEVICE])
@pytest.mark.parametrize("name", WRITE_TESTS)
def test_transcribed_tensor_tests_on_both_routes(name, route):
    msg = hm.run_write_test(name, route)
    assert msg == "", msg


# ---- model check: twin tensors, one per route ----
def same_state(a, b, what):
    ta, tb = a.tuples(), b.tuples()
    for k, (x, y) in enumerate(zip(ta, tb)):
        for u, v in zip(x, y):
            assert (u is None and v is None) or np.array_equal(u, v), f"{what}: layer {fb.grb.TENSOR_LAYERS[k]} differs"
    assert np.array_equal(a.counts(), b.counts()), f"{what}: counters {a.counts()} vs {b.counts()}"
    assert a.edge_count() == b.edge_count(), f"{what}: edge_count"


def test_model_check_twin_tensors():
    rng = np.random.default_rng(2024)
    n = 40
    s0 = rng.integers(0, n, 120)
    d0 = rng.integers(0, n, 120)
    s0 = np.concatenate([s0, s0[:8]])                                    # a few multi-edge pairs in the load
    d0 = np.concatenate([d0, d0[:8]])
    ids0 = np.arange(len(s0))
    ref, dev = hm.Tensor(n, s0, d0, ids0), hm.Tensor(n, s0, d0, ids0)
    edges = [(int(i), int(s), int(d)) for i, s, d in zip(ids0, s0, d0)]    # every edge ever added: removes draw from it
    removed = []
    next_id = len(s0)
    kinds = {"add": 0, "remove": 0, "dup": 0, "fold": 0, "flush": 0}
    steps = 2000
    for step in range(steps):
        r = rng.random()
        if r < 0.45:
            kinds["add"] += 1
            k = int(rng.integers(1, 10))
            batch = []
            for _ in range(k):
                q = rng.random()
                if q < 0.3 and edges:                                    # a pair that has or had edges: promotion of singles
                    _, s, d = edges[int(rng.integers(len(edges)))]
                elif q < 0.45 and removed:                               # re-add over a tombstone, same or a different id
                    i, s, d = removed[int(rng.integers(len(removed)))]
                    if rng.random() < 0.5:
                        batch.append((i, s, d))
                        continue
                else:
                    s, d = int(rng.integers(n)), int(rng.integers(n))
                batch.append((next_id, s, d))
                next_id += 1
            if rng.random() < 0.3:
                batch += batch[: max(1, len(batch) // 2)]                # in-batch duplicates
            ids, ss, ds = zip(*batch)
            ref.add(ss, ds, ids, route=hm.WRITE_REFERENCE)
            dev.add(ss, ds, ids, route=hm.WRITE_DEVICE)
            edges += [(i, s, d) for i, s, d in batch]
        elif r < 0.85:
            kinds["remove"] += 1
            k = int(rng.integers(1, 10))
            rel = [edges[int(rng.integers(len(edges)))] for _ in range(k)]
            if rng.random() < 0.3:                                       # every id a pair has had: demote, then empty
                _, s, d = rel[0]
                rel += [e for e in edges if e[1] == s and e[2] == d]
            if rng.random() < 0.2:
                rel += rel[:2]                                           # repeated ids
            rel = [rel[i] for i in rng.permutation(len(rel))]
            ids, ss, ds = zip(*rel)
            e1 = ref.remove(ids, ss, ds, route=hm.WRITE_REFERENCE)
            e2 = dev.remove(ids, ss, ds, route=hm.WRITE_DEVICE)
            assert set(map(tuple, e1.tolist())) == set(map(tuple, e2.tolist())), f"step {step}: emptied pairs differ"
            removed += rel
        elif r < 0.92:
            kinds["dup"] += 1
            ref, dev = ref.dup(), dev.dup()
        elif r < 0.96:
            kinds["fold"] += 1
            ref.fold_oversized()
            dev.fold_oversized()
        else:
            kinds["flush"] += 1
            ref.flush()
            dev.flush()
        same_state(ref, dev, f"step {step}")
    assert min(kinds.values()) > 0, kinds


# ---- no download of a bulk-loaded base ----
def test_device_route_does_not_download_the_base():
    rng = np.random.default_rng(5)
    n, m = 1 << 16, 400_000
    s, d = rng.integers(0, n, m), rng.integers(0, n, m)
    s[:4000], d[:4000] = s[4000:8000], d[4000:8000]                      # about 1 % multi-edge pairs: remove_all's plan path
    ids = np.arange(m)
    dev, ref = hm.Tensor(n, s, d, ids), hm.Tensor(n, s, d, ids)
    k = 1000
    a_s, a_d = rng.integers(0, n, k), rng.integers(0, n, k)
    a_s[:100], a_d[:100] = s[:100], d[:100]                              # promotions of loaded pairs
    a_id = np.arange(m, m + k)
    r_sel = rng.choice(m, k, replace=False)
    for t, route in ((dev, hm.WRITE_DEVICE), (ref, hm.WRITE_REFERENCE)):
        fb.reset_stats()
        t.add(a_s, a_d, a_id, route=route)
        t.remove(ids[r_sel], s[r_sel], d[r_sel], route=route)
        moved = fb.get_stat("d2h_bytes")
        if route == hm.WRITE_DEVICE:
            # per call: the run count and two totals (24 bytes), at most n 25-byte records and 2n 17-byte me entries
            assert moved <= 2 * (24 + 59 * k), f"device route moved {moved} bytes D2H"
        else:
            assert moved >= 16 * m, f"reference route moved only {moved} bytes D2H: the base was expected to come down"
    same_state(ref, dev, "after the writes")


# ---- adjacency: set_all_dev equals set_all ----
def vm_from(n, rows, cols):
    L = hm.host()
    L.fdbh_vm_from_csr.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p]
    L.fdbh_vm_from_csr.restype = C.c_void_p
    o = np.lexsort((cols, rows))
    rows, cols = np.asarray(rows)[o], np.asarray(cols)[o]
    keep = np.ones(len(rows), bool)
    keep[1:] = (rows[1:] != rows[:-1]) | (cols[1:] != cols[:-1])
    rows, cols = rows[keep], cols[keep]
    p = np.zeros(n + 1, np.uint64)
    np.cumsum(np.bincount(rows, minlength=n), out=p[1:])
    j = cols.astype(np.uint32)
    v = hm.VersionedMatrix.__new__(hm.VersionedMatrix)
    v.L = L
    v.h = L.fdbh_vm_from_csr(n, n, p.ctypes.data, j.ctypes.data)
    assert v.h
    return v


@pytest.mark.parametrize("new", [False, True])
@pytest.mark.parametrize("with_dm", [False, True])
def test_set_all_dev_equals_set_all(new, with_dm):
    rng = np.random.default_rng(11 + 2 * new + with_dm)
    n = 256
    r0, c0 = rng.integers(0, n, 2000), rng.integers(0, n, 2000)
    twins = [vm_from(n, r0, c0), vm_from(n, r0, c0)]
    if with_dm:
        for v in twins:
            for q in range(1000, 1060):                             # tombstones the batch below does not re-set
                v.remove(int(r0[q]), int(c0[q]))
    rows = np.concatenate([r0[:100], r0[1000:1020], rng.integers(0, n, 200), r0[:10]])   # base entries, tombstoned ones, new, repeats
    cols = np.concatenate([c0[:100], c0[1000:1020], rng.integers(0, n, 200), c0[:10]])
    twins[0].set_all(rows, cols, new=new, route=hm.WRITE_REFERENCE)
    twins[1].set_all(rows, cols, new=new, route=hm.WRITE_DEVICE)
    (ca, la), (cb, lb) = twins[0].state(), twins[1].state()
    assert np.array_equal(ca, cb), f"counters {ca} vs {cb}"
    for x, y in zip(la, lb):
        for u, w in zip(x, y):
            assert np.array_equal(u, w)
    assert len(lb[2][0]) > 0 if with_dm else len(lb[2][0]) == 0
