"""Bidirectional variable-length reach: B200_var_len_reach_both (the DISTINCT endpoints of (a)-[*1..k]-(b)) against
B200_var_len_trails in endpoints mode with DISTINCT taken on the host.

Graph: RMAT-20 and RMAT-24 (edge factor 16, seed 1, generated on the device) without self-loops, ids in COO order, one relationship
type loaded by Tensor::bulk_load, then --delta deletes and --delta inserts that stay pending.  Cells: 1, 16, 256 and 1,024 random
non-isolated starts; k = 2, 3, 4 and unbounded.  Each device cell: one warm-up, then the best of --reps calls on the host clock
(the call ends in a device synchronise: its result's entry count is read).  closure_share = 1 - (the same call with min_hops = 0,
which skips the start's own test) / (the call); kernel_ms = the var_len_reach_both family's CUDA-event time (timing on, a separate
call).  The trail enumerator runs on the cells whose walk count over A + A' (sum over the starts of (A + A')^k 1) is at most
--max-trails; its DISTINCT endpoints are compared with the reach's rows.  Prints one JSON line per cell and the card's name and
power limit read in the same run."""
import argparse
import json
import os
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
    except Exception as e:
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scales", default="20,24")
    ap.add_argument("--delta", type=int, default=100_000)
    ap.add_argument("--starts", default="1,16,256,1024")
    ap.add_argument("--ks", default="2,3,4,inf")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-trails", type=float, default=6e7, help="largest walk bound the trail enumerator runs")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("var_len_reach_both.py measures on the GPU: no CUDA device")
    import ctypes as C
    import scipy.sparse as sp
    import falkordb_b200 as fb
    from falkordb_b200 import host_mirror as hm
    from falkordb_b200._lib import lib, U64
    fb.init()
    info = {"card": card(), "delta": a.delta, "rows": []}
    print(json.dumps({"card": info["card"]}), flush=True)
    ks = [None if x == "inf" else int(x) for x in a.ks.split(",")]
    counts = [int(x) for x in a.starts.split(",")]
    for scale in [int(x) for x in a.scales.split(",")]:
        n = 1 << scale
        G = fb.rmat(scale, 16, 1)
        p, j, _ = G.export_csr()
        del G
        rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(p).astype(np.int64))
        cols = j.astype(np.uint64)
        keep = rows != cols
        rows, cols = rows[keep], cols[keep]
        ids = np.arange(len(rows), dtype=np.uint64)
        rng = np.random.default_rng(7)
        gone = rng.choice(len(rows), a.delta, replace=False)
        ns, nd = rng.integers(0, n, a.delta).astype(np.uint64), rng.integers(0, n, a.delta).astype(np.uint64)
        ok = ns != nd
        T = hm.Tensor(n, rows, cols, ids)
        T.remove(ids[gone], rows[gone], cols[gone], route=hm.WRITE_DEVICE)
        T.add(ns[ok], nd[ok], np.arange(len(ids), len(ids) + int(ok.sum()), dtype=np.uint64), route=hm.WRITE_DEVICE)
        Mb = sp.csr_matrix((np.ones(len(rows), np.float32), (rows.astype(np.int64), cols.astype(np.int64))), shape=(n, n))
        Mb = (Mb + Mb.T).tocsr()
        walks = [np.ones(n)]
        for _ in range(4):
            walks.append(Mb @ walks[-1])
        pool = np.nonzero(np.diff(Mb.indptr) > 0)[0]
        del Mb, rows, cols
        L = [T.layers()]
        for k in ks:
            for ns_ in counts:
                st = np.sort(rng.choice(pool, ns_, replace=False)).astype(np.uint64)
                row = {"scale": scale, "k": "inf" if k is None else k, "starts": ns_}

                def call(lo):
                    R = fb.var_len_reach_both(st, L, lo, k)
                    return R, R.nvals()
                call(1)
                best = best0 = 1e30
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    R, nv = call(1)
                    best = min(best, time.perf_counter() - t0)
                    del R
                    t0 = time.perf_counter()
                    R0, nv0 = call(0)
                    best0 = min(best0, time.perf_counter() - t0)
                    del R0
                fb.set_option("timing", 1)
                fb.reset_stats()
                R, nv = call(1)
                ms, nl, by = C.c_double(0), U64(0), U64(0)
                lib().B200_kernel_stats(b"var_len_reach_both", C.byref(ms), C.byref(nl), C.byref(by))
                fb.set_option("timing", 0)
                row.update(pairs=int(nv), ms=best * 1e3, reach_only_ms=best0 * 1e3, closure_share=max(0.0, 1 - best0 / best),
                           kernel_ms=ms.value, kernel_gbs=by.value / (ms.value * 1e6) if ms.value else 0.0,
                           starts_closed=int(nv - (nv0 - ns_)))
                bound = float(walks[4 if k is None else k][st.astype(np.int64)].sum()) if k is not None else float("inf")
                row["walk_bound"] = bound
                if bound <= a.max_trails:
                    fb.var_len_trails(st, L, fb.DIR_BOTH, 1, k, mode="ends")
                    tb = 1e30
                    for _ in range(1 if bound > 1e7 else a.reps):
                        t0 = time.perf_counter()
                        r = fb.var_len_trails(st, L, fb.DIR_BOTH, 1, k, mode="ends")
                        ends = np.unique((np.repeat(np.arange(ns_, dtype=np.uint64), np.diff(r["p"]).astype(np.int64)) << np.uint64(32))
                                         | r["end"].astype(np.uint64))
                        tb = min(tb, time.perf_counter() - t0)
                    I, J, _ = R.extract_tuples()
                    assert np.array_equal(np.unique((I << np.uint64(32)) | J), ends), "reach differs from the trails' DISTINCT ends"
                    row.update(trails=int(r["nout"]), trails_distinct_ms=tb * 1e3, speedup=tb / best)
                else:
                    row["trails"] = "not run"
                del R
                info["rows"].append(row)
                print(json.dumps(row), flush=True)
        del T, L
        fb.lib().B200_pool_trim()
    print(json.dumps({"card": card()}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
