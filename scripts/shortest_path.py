"""shortestPath on the device: the host mirror's shortest_path (one B200_shortest_path call, then one B200_expand_edges call for
the ids) against the reference's route, shortest_path_by_iter (NeighborIter's bidirectional BFS per row and Tensor::get per pair).

Graph: RMAT-20 and RMAT-24 (edge factor 16, seed 1, generated on the device), the edges dealt into 1 or 3 relationship types by
edge index and loaded by Tensor::bulk_load, then --delta deletes and --delta inserts per type that stay pending.  Patterns name
every type: directed (forward layers, then matrix_t backward) and undirected; max_hops 3 and unbounded.  Pairs: 1, 16, 256 and
1,024 random non-isolated pairs, a quarter of them made unreachable by an isolated destination.  Each device cell: one warm-up, then
the best of --reps calls on the host clock (the call ends with its results on the host); kernel_share = the shortest_path family's
CUDA-event time over the same call's host time (timing on, a separate call; the events span the call's device work including the
host's scalar reads between launches); d2h_bytes of one call.  The reference route runs on cells of at most
--ref-pairs pairs; its first call on a tensor (which downloads the bases it reads) is reported apart as ref_cold_ms.  Outputs are
compared whenever both routes ran.  Prints one JSON line per cell and the card's name and power limit read in the same run."""
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
    ap.add_argument("--types", default="1,3")
    ap.add_argument("--delta", type=int, default=100_000)
    ap.add_argument("--pairs", default="1,16,256,1024")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-pairs", type=int, default=16, help="largest batch the reference route runs on")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("shortest_path.py measures on the GPU: no CUDA device")
    import ctypes as C
    import falkordb_b200 as fb
    from falkordb_b200 import host_mirror as hm
    from falkordb_b200._lib import lib, U64
    fb.init()
    info = {"card": card(), "delta": a.delta, "rows": []}
    print(json.dumps({"card": info["card"]}), flush=True)
    for scale in [int(x) for x in a.scales.split(",")]:
        n = 1 << scale
        A = fb.rmat(scale, 16, 1)
        p, j, _ = A.export_csr()
        del A
        rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(p).astype(np.int64))
        cols = j.astype(np.uint64)
        deg = np.bincount(rows.astype(np.int64), minlength=n) + np.bincount(cols.astype(np.int64), minlength=n)
        live, isolated = np.flatnonzero(deg > 0), np.flatnonzero(deg == 0)
        for ntypes in [int(x) for x in a.types.split(",")]:
            rng = np.random.default_rng(scale * 10 + ntypes)
            types, nid = [], len(rows)
            for t in range(ntypes):
                sel = np.arange(t, len(rows), ntypes)
                T = hm.Tensor(n, rows[sel], cols[sel], sel.astype(np.uint64))
                gone = rng.choice(len(sel), min(a.delta, len(sel)), replace=False)
                T.remove(sel[gone].astype(np.uint64), rows[sel][gone], cols[sel][gone], route=hm.WRITE_DEVICE)
                ns, nd = rng.choice(live, a.delta).astype(np.uint64), rng.choice(live, a.delta).astype(np.uint64)
                T.add(ns, nd, np.arange(nid, nid + a.delta, dtype=np.uint64), route=hm.WRITE_DEVICE)
                nid += a.delta
                types.append(T)
            ref_cold = {}
            for directed in (True, False):
                for hi in (3, None):
                    for npairs in [int(x) for x in a.pairs.split(",")]:
                        srcs = rng.choice(live, npairs).astype(np.uint64)
                        dsts = rng.choice(live, npairs).astype(np.uint64)
                        q = npairs // 4
                        if q and len(isolated):
                            dsts[:q] = rng.choice(isolated, q)
                        call = lambda route: hm.shortest_path(None, types, types, srcs, dsts, directed, 1, hi, route=route)
                        dev = call(hm.SP_DEVICE)                     # warm-up
                        best = float("inf")
                        for _ in range(a.reps):
                            t0 = time.perf_counter()
                            dev = call(hm.SP_DEVICE)
                            best = min(best, time.perf_counter() - t0)
                        fb.reset_stats()
                        call(hm.SP_DEVICE)
                        d2h = fb.get_stat("d2h_bytes")
                        fb.set_option("timing", 1)
                        fb.reset_stats()
                        t0 = time.perf_counter()
                        call(hm.SP_DEVICE)
                        timed_ms = (time.perf_counter() - t0) * 1e3
                        ms, nl, by = C.c_double(0), U64(0), U64(0)
                        lib().B200_kernel_stats(b"shortest_path", C.byref(ms), C.byref(nl), C.byref(by))
                        kms = ms.value
                        fb.set_option("timing", 0)
                        row = {"scale": scale, "types": ntypes, "directed": directed, "max_hops": hi, "pairs": npairs,
                               "found": sum(x is not None for x in dev), "dev_ms": round(best * 1e3, 3), "d2h_bytes": int(d2h),
                               "kernel_share": round(kms / timed_ms, 3)}
                        if npairs <= a.ref_pairs:
                            if not ref_cold:
                                t0 = time.perf_counter()
                                call(hm.SP_BY_ITER)
                                ref_cold["ms"] = (time.perf_counter() - t0) * 1e3
                                row["ref_cold_ms"] = round(ref_cold["ms"], 3)
                            t0 = time.perf_counter()
                            ref = call(hm.SP_BY_ITER)
                            row["ref_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
                            row["equal"] = ref == dev
                            assert row["equal"], row
                        info["rows"].append(row)
                        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
