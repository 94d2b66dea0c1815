"""Hop 3's pull under L2 cache policies: which policy keeps the pull's hot gather set in the H100's L2?

Workload: bench.py's chain (RMAT-24, edge factor 16, seed 1, the same seeded source batches as bench.py's rank 0, warm-up batches
included) at 64, 128, 256, 512 and 1,024 sources (W = 1 ... 16).  Per batch, hops 1 and 2 run as in the bench; then hop 3 runs
once per arm, arms alternated, and is timed with CUDA events on the library stream:
  off         : hints = 0 -- plain loads and stores (the kernels as they were before policies)
  streams     : hints = 1, hot_bytes = 0 -- A' col_idx / rowptr, the segment list and the stores of Y evict_first, X evict_normal
  prefix k/8  : hints = 1, hint_streams = 0 -- the first k/8 of the L2 of the packed frontier evict_last, the rest evict_first
  both k/8    : the two together
  default     : the library's defaults
  shuffled    : hints = 0 through a second copy of the graph whose hot-set order is a hash (hot_shuffle = 1): no hot prefix at
                all, so no record is gathered more often in one part of X than in another.  It bounds what residency is worth.
Prints, per source count and arm, the mean over the batches of the per-batch median (over --repeats rounds) of the hop-3 time and
of the bits_pull kernel time, and checks that the hop-3 digests of all arms agree.  Prints one JSON document with the card's
name, power limit and SM clock read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

DEFAULTS = {"hints": -1, "hint_streams": -1, "hot_bytes": -1}


def pull_ms(lib):
    ms, n, b = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    lib.B200_kernel_stats(b"bits_pull", C.byref(ms), C.byref(n), C.byref(b))
    return ms.value


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--sources", default="64,128,256,512,1024")
    ap.add_argument("--batches", type=int, default=13, help="bench.py's --steps + --warmup")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--eighths", default="1,2,3,4,5", help="hot prefixes, in eighths of the L2")
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("pull_l2.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib
    from falkordb_b200.grb import Matrix
    from bench import pick_sources
    from push_gate import card

    fb.init()
    fb.set_option("timing", 1)
    l2 = int(fb.get_stat("l2_bytes"))
    n = 1 << a.scale
    graphs = {}
    for sh in (0, 1):                           # the hot-set order is fixed when the tables are built
        fb.set_option("hot_shuffle", sh)
        graphs[sh] = fb.rmat(a.scale, 16, a.seed)
        graphs[sh].prepare(True)
    fb.set_option("hot_shuffle", 0)
    eighths = [int(k) for k in a.eighths.split(",") if k]
    arms = {"off": (0, {"hints": 0}), "streams": (0, {"hints": 1, "hint_streams": 1, "hot_bytes": 0})}
    arms.update({f"prefix {k}/8": (0, {"hints": 1, "hint_streams": 0, "hot_bytes": l2 * k // 8}) for k in eighths})
    arms.update({f"both {k}/8": (0, {"hints": 1, "hint_streams": 1, "hot_bytes": l2 * k // 8}) for k in eighths})
    arms["default"] = (0, {})
    arms["shuffled"] = (1, {"hints": 0})
    p, _, _ = graphs[0].export_csr()
    deg = np.diff(p.astype(np.int64))
    strm = torch.cuda.ExternalStream(lib().B200_stream())
    L = lib()

    def run_arm(F2, arm):
        g, opts = arms[arm]
        for k, v in {**DEFAULTS, **opts}.items():
            fb.set_option(k, v)
        G = F2[g].dup()
        fb.sync()
        m0 = pull_ms(L)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(strm)
        G.lmxm(graphs[g])
        ev[1].record(strm)
        ev[1].synchronize()
        path = int(fb.get_stat("last_path"))
        return pull_ms(L) - m0, ev[0].elapsed_time(ev[1]), path, tuple(int(x) for x in G.digest())

    doc = {"card": card(), "l2_bytes": l2, "arms": {k: {"graph": "shuffled" if g else "degree order", **v} for k, (g, v) in arms.items()},
           "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "batches": a.batches, "repeats": a.repeats},
           "runs": []}
    for nsrc in [int(s) for s in a.sources.split(",") if s]:
        batches = pick_sources(deg, a.batches, nsrc, a.seed, 0)
        rows = np.arange(nsrc, dtype=np.uint64)
        per = {k: {"hop3": [], "pull": []} for k in arms}
        paths = set()
        for b, src in enumerate(batches):
            for k, v in DEFAULTS.items():
                fb.set_option(k, v)
            F2 = {}
            for g, A in graphs.items():         # hops 1 and 2, as in the bench
                F = Matrix(nsrc, n, bool)
                F.build(rows, src)
                F.lmxm(A)
                F.lmxm(A)
                F2[g] = F
            t = {k: ([], []) for k in arms}
            dg = {}
            for r in range(a.repeats + 1):      # the first round is warm-up
                for arm in arms:
                    pm, h3, path, d = run_arm(F2, arm)
                    paths.add(path)
                    dg[arm] = d
                    if r:
                        t[arm][0].append(pm)
                        t[arm][1].append(h3)
            if len(set(dg.values())) != 1:
                sys.exit(f"{nsrc} sources, batch {b}: the arms' hop-3 digests differ: {dg}")
            for k in arms:
                per[k]["pull"].append(statistics.median(t[k][0]))
                per[k]["hop3"].append(statistics.median(t[k][1]))
            del F2
        run = {"sources": nsrc, "W": (nsrc + 63) // 64, "hop3_paths": sorted(paths),
               "arms": {k: {m: {"mean": round(statistics.fmean(v), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
                            for m, v in d.items()} for k, d in per.items()}}
        doc["runs"].append(run)
        print(f"\n{nsrc} sources (W = {run['W']}), hop-3 paths {run['hop3_paths']}: mean over {a.batches} batches, ms", flush=True)
        base = run["arms"]["off"]["hop3"]["mean"]
        for k, d in run["arms"].items():
            print(f"  {k:12s} hop 3 {d['hop3']['mean']:8.3f} ({d['hop3']['min']:.3f}-{d['hop3']['max']:.3f})"
                  f"  bits_pull {d['pull']['mean']:8.3f}  vs off {d['hop3']['mean'] - base:+.3f}", flush=True)
    doc["card_after"] = card()
    for k, v in DEFAULTS.items():
        fb.set_option(k, v)
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
