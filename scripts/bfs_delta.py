"""algo.BFS over relationship types with pending writes: B200_bfs_delta against the reference's route.

Graph: RMAT-24 (edge factor 16, seed 1) split into T relationship types by a seeded edge hash, for T in --types.  Each type gets
|dp| = |dm| = D for each D in --sizes: dm a seeded random subset of the type's entries, dp seeded random pairs.  Sources: --sources
seeded non-isolated vertices.  Arms, in the same process, alternated source by source:
  (a)  extract : the reference's composition per call -- the union materialised with the public calls (extract(T_1), then
                 set_pattern(<!dm_t> m_t) and set_pattern(dp_t) per further type) into a fresh matrix, then
                 LAGr_BreadthFirstSearch_Extended on it (no transpose mirror: the top-down BFS)
  (b)  delta   : B200_bfs_delta over the types' (m, dp, dm), the bases' mirrors warm
  (b0) first   : B200_bfs_delta on fresh copies of the bases (their mirror and degree table built inside the call); one call
                 per (T, D) row, not alternated
  (c)  control : B200_bfs_ex on the materialised union, prepared once (B200_Matrix_prepare(U, 1)) outside the timing
With --edges, the procedure end to end (csrc/host/algo_bfs.hpp) on a smaller graph (--edges-scale): algo_bfs against
algo_bfs_by_extract over host-mirror Tensors with pending writes, nodes and edges compared.
A call is timed by a host clock around it, ending in a device synchronise.  Every timed call's levels and parents are compared
across (a), (b) and (c); any difference fails the script.  Prints one JSON line per row and one JSON document, with the card's
name, power limit and SM clock read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:                     # the measurement itself needs no nvidia-smi
        return {"error": str(e)}


def spread(v):
    return {"median": round(statistics.median(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--types", default="1,3")
    ap.add_argument("--sizes", default="0,256,100000,1000000")
    ap.add_argument("--sources", type=int, default=16)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--edges", action="store_true", help="also time the procedure end to end through the host mirror")
    ap.add_argument("--edges-scale", type=int, default=18)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("bfs_delta.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib, BfsInfo, P, U64
    from falkordb_b200.grb import Descriptor, Matrix

    fb.init()
    L = lib()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    p, j, _ = A.export_csr()
    del A
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(p.astype(np.int64)))
    cols = j.astype(np.uint64)
    hsh = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F)) ^ np.uint64(a.seed)) >> np.uint64(61)
    live = np.nonzero(np.diff(p))[0]
    rng = np.random.default_rng(a.seed)
    lv = {k: np.empty(n, np.int64) for k in ("a", "b", "c")}
    pr = {k: np.empty(n, np.int64) for k in ("a", "b", "c")}

    def split(T):
        kind = (hsh % np.uint64(T)).astype(np.int8)
        out = []
        for t in range(T):
            sel = np.nonzero(kind == t)[0]
            pt = np.zeros(n + 1, np.uint64)
            np.cumsum(np.bincount(rows[sel].astype(np.int64), minlength=n), out=pt[1:])
            out.append(((pt, j[sel]), sel))
        return out

    def deltas(sel, D):
        dm, dp = Matrix(n, n, bool), Matrix(n, n, bool)
        if D:
            pick = rng.choice(len(sel), size=D, replace=False)
            dm.build(rows[sel][pick], cols[sel][pick])
            dp.build(rng.integers(0, n, D).astype(np.uint64), rng.integers(0, n, D).astype(np.uint64))
        dm.wait(); dp.wait()
        return dp, dm

    def union_by_extract(ops):
        U = Matrix(n, n, bool)
        m, dp, dm = ops[0]
        U.set_pattern(None, m)
        if dm.nvals():
            U.remove_all(dm)
        if dp.nvals():
            U.set_pattern(None, dp)
        for m, dp, dm in ops[1:]:
            U.set_pattern(dm, m, Descriptor.C)
            U.set_pattern(None, dp)
        return U

    def lagr_bfs(U, src):
        """LAGr_BreadthFirstSearch_Extended on U, the graph borrowing U's handle as the reference's procedure lends it"""
        G, h = P(), P(U.h.value)
        fb.check(L.LAGraph_New(C.byref(G), C.byref(h), 1, None))
        vl, vp = P(), P()
        info = L.LAGr_BreadthFirstSearch_Extended(C.byref(vl), C.byref(vp), G, int(src), -1, -1, False, None)
        C.cast(G, C.POINTER(P))[0] = None                  # detach G->A (the first field) before LAGraph_Delete
        L.LAGraph_Delete(C.byref(G), None)
        fb.check(info)
        for v, out in ((vl, lv["a"]), (vp, pr["a"])):
            idx, val, nv = np.empty(n, np.uint64), np.empty(n, np.int64), U64(n)
            fb.check(L.GrB_Vector_extractTuples_INT64(idx.ctypes.data, val.ctypes.data, C.byref(nv), v))
            out.fill(-1)
            out[idx[:nv.value].astype(np.int64)] = val[:nv.value]
            L.GrB_Vector_free(C.byref(v))

    def timed(fn):
        fb.sync()
        t0 = time.perf_counter()
        fn()
        fb.sync()
        return (time.perf_counter() - t0) * 1e3

    def arm_a(ops, src):
        U = union_by_extract(ops)
        lagr_bfs(U, src)
        del U

    def arm_b(ops, src):
        info = BfsInfo()
        arr = lambda xs: (C.c_void_p * len(xs))(*[None if x is None else x.h for x in xs])
        fb.check(L.B200_bfs_delta(arr([o[0] for o in ops]), arr([o[1] for o in ops]), arr([o[2] for o in ops]), len(ops), int(src), -1,
                                  -1, lv["b"].ctypes.data, pr["b"].ctypes.data, 0, C.byref(info)))
        return info

    def arm_c(U, src):
        info = BfsInfo()
        fb.check(L.B200_bfs_ex(U.h, int(src), -1, -1, lv["c"].ctypes.data, pr["c"].ctypes.data, 0, C.byref(info)))
        return info

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "sources": a.sources,
                                        "timing": "host clock around each call, ending in a device synchronise"}, "rows": []}
    src_all = rng.choice(live, a.sources, replace=False)
    for T in [int(s) for s in a.types.split(",")]:
        parts = split(T)
        for D in [int(s) for s in a.sizes.split(",")]:
            bases = [Matrix.import_csr(n, n, pt, jj, None, bool) for (pt, jj), _ in parts]
            ops = [(m,) + deltas(sel, D) for m, (_, sel) in zip(bases, parts)]
            # (b0): the first call on fresh bases builds their mirrors and degree tables inside the call
            b0 = timed(lambda: arm_b(ops, src_all[0]))
            Uc = union_by_extract(ops).prepare(True)
            arm_b(ops, src_all[0]); arm_c(Uc, src_all[0]); arm_a(ops, src_all[0])          # warm every shape
            times = {k: [] for k in "abc"}
            info_b = None
            for s in src_all:
                times["a"].append(timed(lambda: arm_a(ops, s)))
                fb.sync()
                t0 = time.perf_counter()
                info_b = arm_b(ops, s)
                fb.sync()
                times["b"].append((time.perf_counter() - t0) * 1e3)
                times["c"].append(timed(lambda: arm_c(Uc, s)))
                if not (np.array_equal(lv["a"], lv["b"]) and np.array_equal(lv["b"], lv["c"]) and np.array_equal(pr["a"], pr["b"])
                        and np.array_equal(pr["b"], pr["c"])):
                    sys.exit(f"parity: T = {T}, |delta| = {D}, source {s}: levels or parents differ across (a), (b), (c)")
            row = {"types": T, "delta_entries_per_type": D, "call_ms": {k: spread(v) for k, v in times.items()},
                   "first_call_ms_b0": round(b0, 3), "union_nnz": Uc.nvals(),
                   "b_last": {"depth": info_b.depth, "td_levels": info_b.td_levels, "bu_levels": info_b.bu_levels},
                   "levels_parents_identical_a_b_c": True}
            doc["rows"].append(row)
            print(json.dumps(row), flush=True)
            del ops, bases, Uc
        del parts
    if a.edges:
        doc["edges"] = procedure_rows(a, rng)
    doc["card_after"] = card()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


def procedure_rows(a, rng):
    """algo_bfs against algo_bfs_by_extract, want_edges on, over 3 host-mirror Tensors of an RMAT graph with pending writes"""
    import falkordb_b200 as fb
    import falkordb_b200.host_mirror as hm
    import oracle as orc
    n = 1 << a.edges_scale
    A = orc.rmat_csr(a.edges_scale, 16, a.seed)
    r, c, _ = A.tuples()
    kind = rng.integers(0, 3, len(r))
    types, nid = [], 0
    for t in range(3):
        sel = np.nonzero(kind == t)[0]
        ids = np.arange(nid, nid + len(sel), dtype=np.uint64)
        nid += len(sel)
        T = hm.Tensor(n, r[sel], c[sel], ids)
        k = min(10000, len(sel) // 10)
        ns, nd = rng.integers(0, n, k), rng.integers(0, n, k)
        T.add(ns, nd, np.arange(nid, nid + k, dtype=np.uint64))
        nid += k
        gone = rng.choice(len(sel), k, replace=False)
        T.remove(ids[gone], r[sel][gone], c[sel][gone])
        types.append(T)
    srcs = rng.choice(np.nonzero(np.diff(A.p))[0], a.sources, replace=False)
    rows = []
    for named in ((0,), (0, 1, 2)):
        nt = [types[k] for k in named]
        hm.algo_bfs(None, types, nt, srcs[0]); hm.algo_bfs(None, types, nt, srcs[0], route=hm.BFS_BY_EXTRACT)
        times = {"device": [], "by_extract": []}
        for s in srcs:
            for route, key in ((hm.BFS_DEVICE, "device"), (hm.BFS_BY_EXTRACT, "by_extract")):
                fb.sync()
                t0 = time.perf_counter()
                out = hm.algo_bfs(None, types, nt, s, -1, True, route=route)
                times[key].append((time.perf_counter() - t0) * 1e3)
                if key == "device":
                    got = out
                elif not (np.array_equal(got[0], out[0]) and np.array_equal(got[1], out[1])):
                    sys.exit(f"parity: algo_bfs differs from algo_bfs_by_extract, types {named}, source {s}")
        row = {"procedure": f"algo.BFS with edges, RMAT-{a.edges_scale}, {len(named)} named types, pending writes",
               "call_ms": {k: spread(v) for k, v in times.items()}, "nodes_edges_identical": True}
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


if __name__ == "__main__":
    main()
