"""The CSR push of hop 2 in entry order and in destination slices: does finishing one L2-sized slice of Y at a time pay?

Workload: bench.py's chain (RMAT-24, edge factor 16, seed 1, 512 sources per batch, the same seeded batches as bench.py's rank 0,
warm-up batches included).  Hop 1 runs as in the bench; then hops 2 and 3 run from its CSR once per arm, arms alternated:
  entry   : push_slices = 0 through an operand whose relabelled col_idx was never sorted -- the push before slicing existed
  sorted  : push_slices = 1 -- rows of the relabelled col_idx ascending, one slice (the same REDs, adjacent lanes on adjacent records)
  k       : push_slices = k -- k destination slices (--slices; the default -1 is the library's own choice from the L2 size)
Two copies of the graph are prepared, one with push_slices = 0 (unsorted) and one with it on.  Per arm it prints the median, minimum
and maximum over the batches of bits_push ms (B200_kernel_stats) and of the hop 2 + 3 time (CUDA events on the library stream), and
checks that the hop-3 digests agree.  Prints one JSON document with the card's name, power limit and SM clock read in the same run."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def push_ms(lib):
    ms, n, b = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
    lib.B200_kernel_stats(b"bits_push", C.byref(ms), C.byref(n), C.byref(b))
    return ms.value


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--sources", type=int, default=512)
    ap.add_argument("--batches", type=int, default=13, help="bench.py's --steps + --warmup")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--slices", default="-1", help="comma-separated push_slices values to run beside the entry and sorted arms")
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("push_slices.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib
    from falkordb_b200.grb import Matrix
    from bench import pick_sources
    from push_gate import card

    fb.init()
    fb.set_option("timing", 1)
    n = 1 << a.scale
    graphs = {}
    for ps in (0, -1):                          # the tables take their form from push_slices at the time they are built
        fb.set_option("push_slices", ps)
        graphs[ps] = fb.rmat(a.scale, 16, a.seed)
        graphs[ps].prepare(True)
    arms = {"entry": (0, 0), "sorted": (-1, 1)}
    arms.update({f"slices {k}": (-1, int(k)) for k in a.slices.split(",") if k})
    p, _, _ = graphs[0].export_csr()
    deg = np.diff(p.astype(np.int64))
    batches = pick_sources(deg, a.batches, a.sources, a.seed, 0)
    rows = np.arange(a.sources, dtype=np.uint64)
    strm = torch.cuda.ExternalStream(lib().B200_stream())
    L = lib()

    def run_arm(F1, arm):
        g, ps = arms[arm]
        A = graphs[g]
        G = F1.dup()
        fb.set_option("push_slices", ps)
        fb.sync()
        m0 = push_ms(L)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(strm)
        G.lmxm(A)
        path = int(fb.get_stat("last_path"))
        G.lmxm(A)
        ev[1].record(strm)
        ev[1].synchronize()
        return push_ms(L) - m0, ev[0].elapsed_time(ev[1]), path, tuple(int(x) for x in G.digest())

    doc = {"card": card(), "l2_bytes": int(fb.get_stat("l2_bytes")),
           "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "sources": a.sources, "batches": a.batches,
                        "repeats": a.repeats}, "batches": []}
    per = {k: {"push": [], "hop23": []} for k in arms}
    for b, src in enumerate(batches):
        F1 = Matrix(a.sources, n, bool)
        F1.build(rows, src)
        fb.set_option("push_slices", 0)
        F1.lmxm(graphs[0])                      # hop 1, as in the bench
        F1.wait()
        t = {k: ([], []) for k in arms}
        dg = {}
        for r in range(a.repeats + 1):          # the first round is warm-up
            for arm in arms:
                pm, h23, path, d = run_arm(F1, arm)
                if path != 7:
                    sys.exit(f"batch {b}, {arm}: hop 2 took path {path}, not the CSR push")
                dg[arm] = d
                if r:
                    t[arm][0].append(pm)
                    t[arm][1].append(h23)
        if len(set(dg.values())) != 1:
            sys.exit(f"batch {b}: the arms' hop-3 digests differ: {dg}")
        row = {"batch": b, "nnz_F": int(F1.nvals()), "digest": list(dg["entry"]),
               "push_ms": {k: round(statistics.median(v[0]), 3) for k, v in t.items()},
               "hop23_ms": {k: round(statistics.median(v[1]), 3) for k, v in t.items()}}
        for k in arms:
            per[k]["push"].append(row["push_ms"][k])
            per[k]["hop23"].append(row["hop23_ms"][k])
        print(f"batch {b:2d} nnz(F) {row['nnz_F']:7d} | push ms " + " / ".join(f"{k} {row['push_ms'][k]:.3f}" for k in arms) +
              " | hops 2+3 ms " + " / ".join(f"{row['hop23_ms'][k]:.3f}" for k in arms), flush=True)
        doc["batches"].append(row)
        del F1
    doc["summary"] = {k: {m: {"median": round(statistics.median(v), 3), "min": min(v), "max": max(v)} for m, v in d.items()}
                      for k, d in per.items()}
    doc["card_after"] = card()
    fb.set_option("push_slices", -1)
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
