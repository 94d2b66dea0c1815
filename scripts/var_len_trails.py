"""Variable-length trails: B200_var_len_trails against the reference's DFS (fdbh_var_len_trails_dfs, VarLenIterT over
TypesAdjacency on the host mirror's Tensor).

Graph: RMAT-20 (edge factor 16, seed 1) without self-loops, ids in COO order, one relationship type loaded by Tensor::bulk_load
(base built on the device, no host form), then --delta deletes and --delta inserts that stay pending.  Two states:
  cold : a fresh load; the DFS's first row iterator downloads the base (its first call is reported as cold_ms);
  warm : the same tensor after that download (host form present).
Windows *1..2, *1..3, *2..3 (outgoing) and *1..2 bidirectional; modes count, ends (end node + hops) and paths (every edge and
node); 1, 16, 256 and 1,024 random non-isolated starts.  A cell whose last level would hold more than --max-cand candidates (the
walk count M^max 1 over the starts bounds it), or whose output would pass --max-out-gb, is "not run" on both routes; a DFS cell whose estimate (the previous start count's
time, scaled) passes --budget seconds, or whose walk bound passes --max-dfs, is "not run" on the host.  Each device cell: one warm-up, then the best of --reps calls on
the host clock; kernel share = the var_len_trails family's CUDA-event time over the call time (timing on, separate call); d2h
bytes of one call.  Device and DFS outputs are compared whenever both ran (paths mode: list for list).  Prints one JSON line per
cell, the crossover per (window, mode) and the card's name and power limit read in the same run."""
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
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--delta", type=int, default=100_000)
    ap.add_argument("--starts", default="1,16,256,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--budget", type=float, default=30.0, help="seconds one DFS call may take")
    ap.add_argument("--max-cand", type=float, default=2.5e9, help="largest last-level candidate count run")
    ap.add_argument("--max-out-gb", type=float, default=8.0, help="largest host output (bound from the walk count) run")
    ap.add_argument("--max-dfs", type=float, default=2e7, help="largest walk bound the DFS runs")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("var_len_trails.py measures on the GPU: no CUDA device")
    import scipy.sparse as sp
    import falkordb_b200 as fb
    import oracle as orc
    from falkordb_b200 import host_mirror as hm
    from falkordb_b200._lib import lib, U64
    import ctypes as C
    fb.init()
    info = {"card": card(), "scale": a.scale, "delta": a.delta}
    n = 1 << a.scale
    A = orc.rmat_csr(a.scale, 16, 1)
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(A.p))
    cols = A.j.astype(np.uint64)
    keep = rows != cols
    rows, cols = rows[keep], cols[keep]
    ids = np.arange(len(rows), dtype=np.uint64)
    rng = np.random.default_rng(7)
    gone = rng.choice(len(rows), a.delta, replace=False)
    ns, nd = rng.integers(0, n, a.delta).astype(np.uint64), rng.integers(0, n, a.delta).astype(np.uint64)
    ok = ns != nd
    ns, nd = ns[ok], nd[ok]

    def load():
        t = hm.Tensor(n, rows, cols, ids)
        t.remove(ids[gone], rows[gone], cols[gone], route=hm.WRITE_DEVICE)
        t.add(ns, nd, np.arange(len(ids), len(ids) + len(ns), dtype=np.uint64), route=hm.WRITE_DEVICE)
        return t
    M = sp.csr_matrix((np.ones(len(rows)), (rows.astype(np.int64), cols.astype(np.int64))), shape=(n, n))
    walks = [np.ones(n)]
    for _ in range(3):
        walks.append(M @ walks[-1])
    walks_both = [np.ones(n)]
    Mb = M + M.T
    for _ in range(2):
        walks_both.append(Mb @ walks_both[-1])
    deg = np.diff(A.p)
    pool = np.nonzero(deg > 0)[0]
    counts = [int(x) for x in a.starts.split(",")]
    start_sets = {k: np.sort(rng.choice(pool, k, replace=False)).astype(np.uint64) for k in counts}
    windows = [("1..2", fb.DIR_OUT, 1, 2), ("1..3", fb.DIR_OUT, 1, 3), ("2..3", fb.DIR_OUT, 2, 3), ("both 1..2", fb.DIR_BOTH, 1, 2)]
    modes = ["count", "ends", "paths"]

    T = load()
    s0 = start_sets[counts[0]]
    t0 = time.perf_counter()
    hm.var_len_trails([T], s0, fb.DIR_OUT, 1, 1, emit_path=False, route=hm.ROUTE_BY_GET)
    info["cold_dfs_first_call_ms"] = (time.perf_counter() - t0) * 1e3
    Tc = load()                                   # cold: a fresh device-built base for the device route's first call
    fb.reset_stats()
    t0 = time.perf_counter()
    fb.var_len_trails(s0, [Tc.layers()], fb.DIR_OUT, 1, 2, mode="paths")
    info["cold_device_first_call_ms"] = (time.perf_counter() - t0) * 1e3
    info["cold_device_first_call_d2h_bytes"] = fb.get_stat("d2h_bytes")
    del Tc
    print(json.dumps(info), flush=True)

    L = [T.layers()]
    rows_out = []
    for wname, d, lo, hi in windows:
        W = walks_both if d == fb.DIR_BOTH else walks
        for mode in modes:
            prev = None
            for k in counts:
                st = start_sets[k]
                cand = float(W[hi][st.astype(np.int64)].sum())
                row = {"window": wname, "mode": mode, "starts": k, "walk_bound": cand}
                outb = 0 if mode == "count" else cand * (8 + (16 * hi + 4 if mode == "paths" else 0))
                if cand > a.max_cand or outb > a.max_out_gb * 1e9:
                    row["device"] = row["dfs"] = "not run"
                    rows_out.append(row)
                    print(json.dumps(row), flush=True)
                    continue
                fb.var_len_trails(st, L, d, lo, hi, mode=mode)
                best = 1e30
                for _ in range(a.reps):
                    fb.reset_stats()
                    t0 = time.perf_counter()
                    r = fb.var_len_trails(st, L, d, lo, hi, mode=mode)
                    best = min(best, time.perf_counter() - t0)
                    d2h = fb.get_stat("d2h_bytes")
                fb.set_option("timing", 1)
                fb.reset_stats()
                t0 = time.perf_counter()
                fb.var_len_trails(st, L, d, lo, hi, mode=mode)
                wall = time.perf_counter() - t0
                ms, nl, by = C.c_double(0), U64(0), U64(0)
                lib().B200_kernel_stats(b"var_len_trails", C.byref(ms), C.byref(nl), C.byref(by))
                kms, kbytes = ms.value, by.value
                fb.set_option("timing", 0)
                row.update(trails=int(r["nout"]), device_ms=best * 1e3, trails_per_s=r["nout"] / best, d2h_bytes=int(d2h),
                           kernel_share=kms / (wall * 1e3), kernel_gbs=kbytes / (kms * 1e6) if kms else 0.0)
                est = prev[1] * k / prev[0] if prev else 0.0
                if est > a.budget or cand > a.max_dfs:
                    row["dfs"] = "not run"
                else:
                    t0 = time.perf_counter()
                    w = hm.var_len_trails([T], st, d, lo, hi, emit_path=(mode == "paths"), route=hm.ROUTE_BY_GET)
                    h = time.perf_counter() - t0
                    prev = (k, h)
                    row.update(dfs_ms=h * 1e3, speedup=h / best)
                    assert np.array_equal(w["p"], r["p"]), "trail counts differ"
                    if mode != "count":
                        assert np.array_equal(w["end"], r["end"].astype(np.uint64)) and np.array_equal(w["hops"], r["hops"].astype(np.uint64))
                    if mode == "paths":
                        assert np.array_equal(w["edges"], r["edges"]) and np.array_equal(w["nodes"], r["nodes"].astype(np.uint64))
                rows_out.append(row)
                print(json.dumps(row), flush=True)
    cross = {}
    for r in rows_out:
        key = f"{r['window']} {r['mode']}"
        if "speedup" in r and r["speedup"] >= 1 and key not in cross:
            cross[key] = r["starts"]
    info["crossover_starts"] = cross
    info["rows"] = rows_out
    print(json.dumps({"crossover_starts": cross, "card": info["card"]}), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
