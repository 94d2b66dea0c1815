"""Named-edge, incoming and bidirectional expansion: B200_expand_edges against the routes it replaces.

Graph: RMAT-24 (edge factor 16, seed 1) with edge ids in COO order, plus a share (--multi) of pairs carrying a second edge (new
ids), split into T relationship types by a seeded edge hash, for T in --types.  Each type is a host-mirror Tensor loaded by
Tensor::bulk_load (base built on the device, no host form).  State "clean" is measured first; then every type gets --delta new
edges (random pairs, Tensor::set_all_from_slices) and --delta deleted edges (Tensor::remove_all), which stay pending, and state
"dirty" is measured.  Source sets: 1 source of median out-degree, the top hub, 1,024 random non-isolated sources.  Directions
OUT and BOTH.  Arms, alternated --reps times after one warm-up call each:
  (a) by_get   : expand_edges_by_get, expand_row's loops over Tensor::get (host mirror).  The first call on the fresh tensors
                 downloads every base (GrB_Matrix_extractElement on a base without host form): reported apart as cold_ms.
  (b) traverse : today's bind_edge route, B200_traverse_batch_union for the pairs, then a Tensor::get per pair (OUT, FIRST only)
  (c) device   : B200_expand_edges (EDGES_ALL and EDGES_FIRST)
Outputs of (a) and (c), and of (b) and (c) FIRST, are compared on every row; any difference fails the script.  A call is timed on
the host clock around the whole call, which ends in a device synchronise.  edge_expand GB/s is the kernel family's compulsory
bytes (edges.cu) over its CUDA-event time in a separate call with timing on, with its fraction of 3.35 TB/s.  Prints one JSON
line per row and one JSON document, with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_GBS = 3350.0


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:                     # the measurement itself needs no nvidia-smi
        return {"error": str(e)}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--types", default="1,3")
    ap.add_argument("--delta", type=int, default=1_000_000)
    ap.add_argument("--multi", type=float, default=0.01, help="share of pairs that get a second edge")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("edge_expand.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200 import host_mirror as hm
    from falkordb_b200._lib import lib
    import ctypes as C

    fb.init()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    p, j, _ = A.export_csr()
    del A
    deg = np.diff(p.astype(np.int64))
    rows = np.repeat(np.arange(n, dtype=np.uint64), deg)
    cols = j.astype(np.uint64)
    del j
    ids = np.arange(len(cols), dtype=np.uint64)
    rng = np.random.default_rng(a.seed)
    extra = rng.choice(len(cols), int(a.multi * len(cols)), replace=False)
    rows = np.concatenate([rows, rows[extra]])
    cols = np.concatenate([cols, cols[extra]])
    ids = np.concatenate([ids, np.arange(len(ids), len(ids) + len(extra), dtype=np.uint64)])
    next_id = len(ids)
    hsh = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F)) ^ np.uint64(a.seed)) >> np.uint64(61)
    live = np.nonzero(deg)[0]
    med = live[np.argsort(deg[live], kind="stable")[len(live) // 2]]
    srcsets = (("1 source, median degree", np.array([med], np.uint64)), ("1 source, top hub", np.array([np.argmax(deg)], np.uint64)),
               ("1024 sources", rng.choice(live, 1024, replace=False).astype(np.uint64)))

    def timed(f):
        t0 = time.perf_counter()
        out = f()
        return (time.perf_counter() - t0) * 1e3, out

    def same(x, y):
        return all(np.array_equal(np.asarray(u, np.uint64), np.asarray(v, np.uint64)) for u, v in zip(x, y))

    def kernel(src, lays, dir, mode):
        fb.set_option("timing", 1)
        lib().B200_reset_stats()
        fb.expand_edges(src, lays, dir, mode)
        ms, nl, by = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
        lib().B200_kernel_stats(b"edge_expand", C.byref(ms), C.byref(nl), C.byref(by))
        fb.set_option("timing", 0)
        return ms.value, by.value

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}, ids in COO order, "
                                                 f"{a.multi:.0%} of pairs with a second edge", "delta_per_type": a.delta,
                                        "reps": a.reps, "timing": "host clock around each call (ends in a device sync)"},
           "rows": []}
    for T in [int(s) for s in a.types.split(",")]:
        kind = (hsh % np.uint64(T)).astype(np.int8)
        tensors, sels = [], []
        for t in range(T):
            sel = np.nonzero(kind == t)[0]
            tensors.append(hm.Tensor(n, rows[sel], cols[sel], ids[sel]))
            sels.append(sel)
        cold = None
        for state in ("clean", "dirty"):
            if state == "dirty":
                for t, x in enumerate(tensors):
                    na, nb = rng.integers(0, n, a.delta).astype(np.uint64), rng.integers(0, n, a.delta).astype(np.uint64)
                    x.add(na, nb, np.arange(next_id, next_id + a.delta, dtype=np.uint64))
                    next_id += a.delta
                    gone = rng.choice(sels[t], a.delta, replace=False)
                    x.remove(ids[gone], rows[gone], cols[gone])
            lays = [x.layers() for x in tensors]
            for name, src in srcsets:
                for dir in (fb.DIR_OUT, fb.DIR_BOTH):
                    arms = {("c", fb.EDGES_ALL): lambda: fb.expand_edges(src, lays, dir, fb.EDGES_ALL),
                            ("c", fb.EDGES_FIRST): lambda: fb.expand_edges(src, lays, dir, fb.EDGES_FIRST),
                            ("a", fb.EDGES_ALL): lambda: hm.expand_edges(tensors, src, dir, fb.EDGES_ALL, route=hm.ROUTE_BY_GET),
                            ("a", fb.EDGES_FIRST): lambda: hm.expand_edges(tensors, src, dir, fb.EDGES_FIRST, route=hm.ROUTE_BY_GET)}
                    if dir == fb.DIR_OUT:
                        arms[("b", fb.EDGES_FIRST)] = lambda: hm.expand_edges(tensors, src, dir, fb.EDGES_FIRST,
                                                                              route=hm.ROUTE_TRAVERSE_GET)
                    outs = {}
                    for k, f in arms.items():
                        ms, outs[k] = timed(f)
                        if cold is None and k[0] == "a":
                            cold = ms             # the first Tensor::get on these tensors: every base comes to the host
                    times = {k: [] for k in arms}
                    for _ in range(a.reps):
                        for k, f in arms.items():
                            ms, out = timed(f)
                            times[k].append(ms)
                            if not same(out, outs[k]):
                                sys.exit(f"{k} is not deterministic ({T} types, {state}, {name}, dir {dir})")
                    for mode in (fb.EDGES_ALL, fb.EDGES_FIRST):
                        if not same(outs[("a", mode)], outs[("c", mode)]):
                            sys.exit(f"parity: by_get differs from the device ({T} types, {state}, {name}, dir {dir}, mode {mode})")
                    if ("b", fb.EDGES_FIRST) in outs and not same(outs[("b", fb.EDGES_FIRST)], outs[("c", fb.EDGES_FIRST)]):
                        sys.exit(f"parity: the traversal-then-get route differs from the device ({T} types, {state}, {name})")
                    kms, kbytes = kernel(src, lays, dir, fb.EDGES_ALL)
                    entries = {mode: int(len(outs[("c", mode)][2])) for mode in (fb.EDGES_ALL, fb.EDGES_FIRST)}
                    arm_name = {"a": "by_get", "b": "traverse_get", "c": "device"}
                    med_ms = {f"{arm_name[k[0]]}_{'all' if k[1] == 0 else 'first'}": round(statistics.median(v), 3)
                              for k, v in times.items()}
                    row = {"types": T, "state": state, "sources": name, "dir": "OUT" if dir == fb.DIR_OUT else "BOTH",
                           "entries_all": entries[fb.EDGES_ALL], "entries_first": entries[fb.EDGES_FIRST], "ms": med_ms,
                           "entries_per_s_all": {arm_name[k[0]]: round(entries[k[1]] / (statistics.median(v) / 1e3))
                                                 for k, v in times.items() if k[1] == fb.EDGES_ALL},
                           "edge_expand_kernel_ms": round(kms, 4), "edge_expand_bytes": kbytes,
                           "edge_expand_GBps": round(kbytes / kms / 1e6, 1) if kms else None,
                           "edge_expand_frac_of_3_35TBps": round(kbytes / kms / 1e6 / HBM_GBS, 3) if kms else None,
                           "parity": True}
                    doc["rows"].append(row)
                    print(json.dumps(row), flush=True)
        doc.setdefault("by_get_cold_first_call_ms", {})[str(T)] = round(cold, 1)
        print(json.dumps({"types": T, "by_get_cold_first_call_ms": round(cold, 1)}), flush=True)
        del tensors, lays
    doc["card_after"] = card()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
