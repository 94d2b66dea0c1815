"""Dirty 3-hop chain: what pending writes cost a traversal, and what the fused delta_lmxm saves.

Workload: RMAT-24 (edge factor 16, seed 1), 3 hops, a fresh batch of 512 random non-isolated sources every step.  Every hop's
operand is (m, dp, dm) with |dp| = |dm| = D for each D in --sizes: dm is a seeded random subset of m's entries, dp seeded random
pairs (the construction of bench.py's delta arm).  Three arms, in the same process, alternated step by step:
  (a) clean : F <- F * m per hop (GrB_mxm, what B200_traverse_batch runs per hop), on m alone
  (b) composed : the reference's delta_lmxm, three GrB_mxm plus an eWiseAdd per hop (Matrix.delta_lmxm)
  (c) fused : B200_Matrix_delta_lmxm per hop (what B200_traverse_batch_delta runs per hop)
A step is the 3-hop chain on a device-resident frontier, timed with CUDA events on the library stream; the one-call entries add
the same host hand-off to (a) and (c).  Per size: the median over --steps steps after --warmup, for each of --repeats runs.
The digests of (b) and (c) are compared after every timed step; any difference fails the script.  A separate pass with kernel
timing on reports the fused kernels' achieved bandwidth ("bits_delta": 12 nnz(delta) + 16 W nnz(delta) bytes per launch).
Prints one JSON document, with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

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


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--nsrc", type=int, default=512)
    ap.add_argument("--hops", type=int, default=3)
    ap.add_argument("--sizes", default="256,4500,100000,1000000")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("delta_chain.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib
    from falkordb_b200.grb import Matrix

    fb.init()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    A.prepare(True)
    p, j, _ = A.export_csr()
    live = np.nonzero(np.diff(p))[0]
    strm = torch.cuda.ExternalStream(lib().B200_stream())
    rng = np.random.default_rng(a.seed)

    def deltas(D):
        pick = np.sort(rng.choice(len(j), size=D, replace=False))
        dm = Matrix(n, n, bool)
        dm.build((np.searchsorted(p, pick, side="right") - 1).astype(np.uint64), j[pick].astype(np.uint64))
        dp = Matrix(n, n, bool)
        dp.build(rng.integers(0, n, D).astype(np.uint64), rng.integers(0, n, D).astype(np.uint64))
        dm.wait(); dp.wait()
        return dp, dm

    def step(arm, src, dp, dm):
        """one chain; returns (ms, F)"""
        F = Matrix(len(src), n, bool)
        F.build(np.arange(len(src)), src)
        fb.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(strm)
        for _ in range(a.hops):
            if arm == "a":
                F.lmxm(A)
            elif arm == "b":
                F.delta_lmxm(A, dp, dm)
            else:
                F.delta_lmxm_fused(A, dp, dm)
        e1.record(strm)
        e1.synchronize()
        return e0.elapsed_time(e1), F

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "nsrc": a.nsrc, "hops": a.hops,
                                        "steps": a.steps, "warmup": a.warmup, "repeats": a.repeats}, "sizes": []}
    for D in [int(s) for s in a.sizes.split(",")]:
        dp, dm = deltas(D)
        runs = {"a": [], "b": [], "c": []}
        for r in range(a.repeats):
            times = {"a": [], "b": [], "c": []}
            for s in range(a.warmup + a.steps):
                src = rng.choice(live, a.nsrc, replace=False)
                dg = {}
                for arm in ("a", "b", "c"):
                    ms, F = step(arm, src, dp, dm)
                    if s >= a.warmup:
                        times[arm].append(ms)
                        if arm != "a":
                            dg[arm] = F.digest()
                    del F
                if s >= a.warmup and not np.array_equal(dg["b"], dg["c"]):
                    sys.exit(f"parity: |delta| = {D}, repeat {r}, step {s}: composed {dg['b']} != fused {dg['c']}")
            for arm in runs:
                runs[arm].append(statistics.median(times[arm]))
        # kernel time of the fused delta passes, in a pass of its own (events around every launch)
        fb.set_option("timing", 1)
        fb.reset_stats()
        for _ in range(3):
            step("c", rng.choice(live, a.nsrc, replace=False), dp, dm)
        import ctypes as C
        ms, nl, by = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
        lib().B200_kernel_stats(b"bits_delta", C.byref(ms), C.byref(nl), C.byref(by))
        fb.set_option("timing", 0)
        row = {"delta_entries": D,
               "step_ms_median_per_repeat": {k: [round(v, 3) for v in vs] for k, vs in runs.items()},
               "step_ms": {k: round(statistics.median(vs), 3) for k, vs in runs.items()},
               "bits_delta": {"launches": nl.value, "ms": round(ms.value, 4), "bytes": by.value,
                              "GB_per_s": round(by.value / (ms.value * 1e-3) / 1e9, 1) if ms.value > 0 else None},
               "digest_parity_b_c": True}
        row["fused_faster_than_composed"] = row["step_ms"]["c"] < row["step_ms"]["b"]
        doc["sizes"].append(row)
        print(json.dumps(row), flush=True)
        del dp, dm
    doc["card_after"] = card()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
