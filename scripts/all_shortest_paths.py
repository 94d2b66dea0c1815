"""allShortestPaths on the device: the host mirror's all_shortest_paths (a counting B200_all_shortest_paths call, then one call that
fills every path) against the reference's route, all_shortest_paths_by_iter (expand_row per row over TypesAdjacency: a FIFO BFS with
one row-iterator seek per type and direction per visited node, then the DFS backtrack).

Graph: RMAT-20 and RMAT-24 (edge factor 16, seed 1, generated on the device), the edges dealt into 1 or 3 relationship types by
edge index and loaded by Tensor::bulk_load, then --delta deletes and --delta inserts per type that stay pending (0 and 10^4 by
default).  Patterns name every type, outgoing and bidirectional, unbounded.  Pairs: 1, 16 and 1,024 reachable pairs with at most
--max-count shortest paths each (drawn from random non-isolated pairs by a counting call, so that both routes can list every
path).  Each device cell: one warm-up, then the best of --reps calls on the host clock (the call ends with every path on the
host); d2h_bytes of one call.  The reference route runs on cells of at most --ref-pairs pairs; its first call on a tensor set
(which downloads the bases it reads) is reported apart as ref_cold_ms.  Outputs are compared whenever both routes ran.  Prints one
JSON line per cell and the card's name and power limit read in the same run."""
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
    ap.add_argument("--deltas", default="0,10000")
    ap.add_argument("--pairs", default="1,16,1024")
    ap.add_argument("--max-count", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ref-pairs", type=int, default=16, help="largest batch the reference route runs on")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("all_shortest_paths.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200 import host_mirror as hm
    fb.init()
    info = {"card": card(), "rows": []}
    print(json.dumps({"card": info["card"]}), flush=True)
    for scale in [int(x) for x in a.scales.split(",")]:
        n = 1 << scale
        A = fb.rmat(scale, 16, 1)
        p, j, _ = A.export_csr()
        del A
        rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(p).astype(np.int64))
        cols = j.astype(np.uint64)
        deg = np.bincount(rows.astype(np.int64), minlength=n) + np.bincount(cols.astype(np.int64), minlength=n)
        live = np.flatnonzero(deg > 0)
        for ntypes in [int(x) for x in a.types.split(",")]:
            for delta in [int(x) for x in a.deltas.split(",")]:
                rng = np.random.default_rng(scale * 100 + ntypes * 10 + (delta > 0))
                types, nid = [], len(rows)
                for t in range(ntypes):
                    sel = np.arange(t, len(rows), ntypes)
                    T = hm.Tensor(n, rows[sel], cols[sel], sel.astype(np.uint64))
                    if delta:
                        gone = rng.choice(len(sel), min(delta, len(sel)), replace=False)
                        T.remove(sel[gone].astype(np.uint64), rows[sel][gone], cols[sel][gone], route=hm.WRITE_DEVICE)
                        ns, nd = rng.choice(live, delta).astype(np.uint64), rng.choice(live, delta).astype(np.uint64)
                        T.add(ns, nd, np.arange(nid, nid + delta, dtype=np.uint64), route=hm.WRITE_DEVICE)
                        nid += delta
                    types.append(T)
                layers = [t.layers() for t in types]
                ref_cold = {}
                for directed in (True, False):
                    d = fb.DIR_OUT if directed else fb.DIR_BOTH
                    cs, cd = rng.choice(live, 8192).astype(np.uint64), rng.choice(live, 8192).astype(np.uint64)
                    c = fb.all_shortest_paths(cs, cd, layers, d, edge_capacity=0)["count"]
                    ok = np.flatnonzero((c > 0) & (c <= a.max_count))
                    for npairs in [int(x) for x in a.pairs.split(",")]:
                        pick = ok[rng.integers(0, len(ok), npairs)]
                        srcs, dsts = cs[pick], cd[pick]
                        call = lambda route: hm.all_shortest_paths(types, types, srcs, dsts, directed, None, route=route)
                        dev = call(hm.ASP_DEVICE)                    # warm-up
                        best = float("inf")
                        for _ in range(a.reps):
                            t0 = time.perf_counter()
                            dev = call(hm.ASP_DEVICE)
                            best = min(best, time.perf_counter() - t0)
                        fb.reset_stats()
                        call(hm.ASP_DEVICE)
                        row = {"scale": scale, "types": ntypes, "delta": delta, "directed": directed, "pairs": npairs,
                               "paths": sum(len(x) for x in dev), "edges": sum(len(e) for x in dev for e, _ in x),
                               "dev_ms": round(best * 1e3, 3), "d2h_bytes": int(fb.get_stat("d2h_bytes"))}
                        if npairs <= a.ref_pairs:
                            if not ref_cold:
                                t0 = time.perf_counter()
                                call(hm.ASP_BY_ITER)
                                ref_cold["ms"] = (time.perf_counter() - t0) * 1e3
                                row["ref_cold_ms"] = round(ref_cold["ms"], 3)
                            t0 = time.perf_counter()
                            ref = call(hm.ASP_BY_ITER)
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
