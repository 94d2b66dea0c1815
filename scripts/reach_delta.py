"""Variable-length reach over a relationship tensor with pending writes: what the exact dirty hop costs against today's routes.

Workload: RMAT-24 (edge factor 16, seed 1), max_hops = 3, a fresh batch of 512 random non-isolated sources every step.  The operand
is (m, dp, dm) with |dp| = |dm| = D for each D in --sizes: dm is a seeded random subset of m's entries, dp seeded random pairs
(the construction of delta_chain.py).  Three arms, in the same process, alternated step by step:
  (a) clean        : B200_reach_batch on the prepared m alone
  (b) materialised : (m \\ dm) u dp written to a fresh matrix (GrB_eWiseAdd under the complemented dm mask, then with dp), its
                     transpose mirror and pull tables built (B200_Matrix_prepare), then B200_reach_batch on it -- all inside the step
  (c) delta        : B200_reach_batch_delta over (m, dp, dm)
A step is one call, timed with CUDA events on the library stream.  Per size: the median over --steps steps after --warmup.  The
digests of (b) and (c) are compared after every timed step; any difference fails the script.  A separate pass with kernel timing
on reports the repair kernel's achieved bandwidth ("bits_repair"), and the repair volume sum over the columns of dm of
indeg_m(j), as a share of nnz(m) (what a full pull gathers).  Prints one JSON document, with the card's name, power limit and SM
clock read in the same run."""
import argparse
import ctypes as C
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
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("reach_delta.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib
    from falkordb_b200.grb import Descriptor, Matrix

    fb.init()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    A.prepare(True)
    p, j, _ = A.export_csr()
    live = np.nonzero(np.diff(p))[0]
    indeg = np.bincount(j, minlength=n)
    strm = torch.cuda.ExternalStream(lib().B200_stream())
    rng = np.random.default_rng(a.seed)

    def deltas(D):
        pick = np.sort(rng.choice(len(j), size=D, replace=False))
        dm = Matrix(n, n, bool)
        dm.build((np.searchsorted(p, pick, side="right") - 1).astype(np.uint64), j[pick].astype(np.uint64))
        dp = Matrix(n, n, bool)
        dp.build(rng.integers(0, n, D).astype(np.uint64), rng.integers(0, n, D).astype(np.uint64))
        dm.wait(); dp.wait()
        share = float(indeg[np.unique(j[pick])].sum()) / len(j)
        return dp, dm, share

    def step(arm, src, dp, dm):
        """one reach; returns (ms, R, levels)"""
        fb.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(strm)
        if arm == "a":
            R, lv = fb.reach_batch(src, A, a.hops)
        elif arm == "b":
            E = Matrix(n, n, bool)
            E.element_wise_add(dm, A, A, Descriptor.RC)          # E<!dm, replace> = m
            E.element_wise_add(None, E, dp)
            E.prepare(True)
            R, lv = fb.reach_batch(src, E, a.hops)
            del E
        else:
            R, lv = fb.reach_batch(src, [A], a.hops, deltas=[(dp, dm)])
        e1.record(strm)
        e1.synchronize()
        return e0.elapsed_time(e1), R, lv

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "nsrc": a.nsrc,
                                        "max_hops": a.hops, "steps": a.steps, "warmup": a.warmup}, "sizes": []}
    for D in [int(s) for s in a.sizes.split(",")]:
        dp, dm, share = deltas(D)
        times = {"a": [], "b": [], "c": []}
        for s in range(a.warmup + a.steps):
            src = rng.choice(live, a.nsrc, replace=False)
            dg = {}
            for arm in ("a", "b", "c"):
                ms, R, lv = step(arm, src, dp, dm)
                if s >= a.warmup:
                    times[arm].append(ms)
                    if arm != "a":
                        dg[arm] = (tuple(R.digest().tolist()), lv)
                del R
            if s >= a.warmup and dg["b"] != dg["c"]:
                sys.exit(f"parity: |delta| = {D}, step {s}: materialised {dg['b']} != delta {dg['c']}")
        fb.set_option("timing", 1)
        fb.reset_stats()
        for _ in range(3):
            step("c", rng.choice(live, a.nsrc, replace=False), dp, dm)
        ms, nl, by = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
        lib().B200_kernel_stats(b"bits_repair", C.byref(ms), C.byref(nl), C.byref(by))
        fb.set_option("timing", 0)
        med = {k: round(statistics.median(v), 3) for k, v in times.items()}
        row = {"delta_entries": D, "step_ms": med, "step_ms_min_max": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
               "bits_repair": {"launches": nl.value, "ms_per_call": round(ms.value / 3, 4), "bytes_per_call": by.value // 3,
                               "GB_per_s": round(by.value / (ms.value * 1e-3) / 1e9, 1) if ms.value > 0 else None},
               "repair_share_of_nnz": round(share, 4), "digest_parity_b_c": True,
               "delta_faster_than_materialised": med["c"] < med["b"]}
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
