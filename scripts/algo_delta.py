"""algo.pageRank, algo.WCC and algo.labelPropagation over relationship types with pending writes: the procedures' device route
(one B200_adjacency_delta call, csrc/host/algo_procs.hpp) against the reference's route (algo_proc_by_extract), end to end through
the host mirror.

Graph: RMAT-S (--scale, edge factor 16, seed 1) loaded into T host-mirror relationship Tensors (GRAPH.BULK's device-side load) split
by a seeded edge hash, for T in --types.  Each type then gets D pending deletes (Tensor::remove_all of seeded random edges) and D
pending inserts (Tensor::set_all_from_slices of seeded random pairs) for each D in --sizes.  Every type is named in the call.  Label
filters: seeded label matrices holding --labels fractions of the vertices; "all" is the unfiltered call (no label: the matrix of
every node, which is also what pageRank runs on when its label covers every node).  Arms, alternated call by call in one process:
  extract : algo_proc_by_extract -- unfiltered, the types' extracts and their eWiseAdd (with the transpose and one more eWiseAdd
            for WCC / CDLP), dup + resize; filtered, the walk over every edge of every type through a host hash map and one
            GxB_Matrix_build_Scalar.  Then the LAGraph call and the output loop.
  device  : algo_proc -- one B200_adjacency_delta call over the types' (m, dp, dm), then the same LAGraph call and output loop.
  builder : B200_adjacency_delta alone on the same operands (the part of `device` that replaces the reference's build).
A call is timed by a host clock around it, ending in a device synchronise.  The node and value columns of every timed device and
extract call are compared; any difference fails the script.  Prints one JSON line per row and one JSON document, with the card's
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
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--types", default="1,3")
    ap.add_argument("--sizes", default="0,10000,1000000")
    ap.add_argument("--labels", default="0.01,0.1,all")
    ap.add_argument("--procs", default="pagerank,wcc,cdlp")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("algo_delta.py measures on the GPU; no CUDA device is visible")
    import falkordb_b200 as fb
    import falkordb_b200.host_mirror as hm
    from falkordb_b200._lib import lib, check, P
    fb.init()
    dev = card()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    p, j, _ = A.export_csr()
    del A
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(p.astype(np.int64)))
    cols = j.astype(np.uint64)
    del p, j
    h = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F))) >> np.uint64(32)
    rng = np.random.default_rng(a.seed)
    fracs = [x for x in a.labels.split(",")]
    label_sets, kept = {}, {}
    for f in fracs:
        if f == "all":
            continue
        vs = np.sort(rng.choice(n, max(1, int(float(f) * n)), replace=False))
        L = hm.VersionedMatrix(n)
        for v in vs.tolist():
            L.set(v, v)
        label_sets[f], kept[f] = L, vs.astype(np.uint64)
    adj = hm.VersionedMatrix(n)        # not walked: every type is named
    fns = {"pagerank": hm.algo_pagerank, "wcc": hm.algo_wcc, "cdlp": hm.algo_cdlp}
    results = []
    for ntypes in [int(x) for x in a.types.split(",")]:
        kind = h % np.uint64(ntypes)
        for D in [int(x) for x in a.sizes.split(",")]:
            types, next_id = [], 0
            for t in range(ntypes):
                sel = np.nonzero(kind == t)[0]
                ids = np.arange(next_id, next_id + len(sel), dtype=np.uint64)
                next_id += len(sel)
                T = hm.Tensor(n, rows[sel], cols[sel], ids)
                if D:
                    pick = rng.choice(len(sel), D, replace=False)
                    T.remove(ids[pick], rows[sel][pick], cols[sel][pick])
                    T.add(rng.integers(0, n, D), rng.integers(0, n, D), np.arange(next_id, next_id + D, dtype=np.uint64))
                    next_id += D
                types.append(T)
            layers = [T.layers() for T in types]
            arr = lambda k: (C.c_void_p * ntypes)(*[ls[k] for ls in layers])
            for proc in a.procs.split(","):
                for f in fracs:
                    labels = [] if f == "all" else [label_sets[f]]
                    t_dev, t_ext, t_bld = [], [], []
                    for rep in range(a.reps + 1):             # the first round warms every shape and is not recorded
                        for arm in ("device", "extract", "builder"):
                            torch.cuda.synchronize()
                            t0 = time.perf_counter()
                            if arm == "builder":
                                M = P()
                                if f == "all":
                                    check(lib().B200_adjacency_delta(C.byref(M), arr(0), arr(1), arr(2), ntypes, n, None, 0,
                                                                     0 if proc == "pagerank" else 1))
                                else:
                                    check(lib().B200_adjacency_delta(C.byref(M), arr(0), arr(1), arr(2), ntypes, n,
                                                                     kept[f].ctypes.data, len(kept[f]), 0 if proc == "pagerank" else 1))
                                torch.cuda.synchronize()
                                dt = time.perf_counter() - t0
                                lib().GrB_Matrix_free(C.byref(M))
                            else:
                                out = fns[proc](adj, types, types, labels, n, (),
                                                route=hm.ALGO_DEVICE if arm == "device" else hm.ALGO_BY_EXTRACT)
                                torch.cuda.synchronize()
                                dt = time.perf_counter() - t0
                                if arm == "device":
                                    got = out
                                else:
                                    if not (np.array_equal(got[0], out[0]) and np.array_equal(got[1], out[1])):
                                        sys.exit(f"{proc} T={ntypes} D={D} label={f}: the routes differ")
                            if rep:
                                {"device": t_dev, "extract": t_ext, "builder": t_bld}[arm].append(1e3 * dt)
                    row = {"proc": proc, "types": ntypes, "pending_per_type": D, "label": f, "rows_out": int(len(got[0])),
                           "extract_ms": spread(t_ext), "device_ms": spread(t_dev), "builder_ms": spread(t_bld), "equal": True}
                    print(json.dumps(row), flush=True)
                    results.append(row)
            del types, layers
    doc = {"card": dev, "scale": a.scale, "edge_factor": 16, "reps": a.reps, "rows": results}
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(doc, fh, indent=1)


if __name__ == "__main__":
    main()
