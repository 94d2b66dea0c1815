"""Hop 2 of the bench chain three ways: where the CSR push's gate belongs.

Workload: bench.py's chain (RMAT-24, edge factor 16, seed 1, 512 sources per batch, the same seeded batches as bench.py's rank 0,
warm-up batches included).  Hop 1 runs as in the bench (row-wise; its result is a CSR).  Then hop 2 runs from that CSR three ways,
each followed by hop 3 under the default options, since the form hop 2 leaves decides hop 3's preparation:
  csr  : csr_push = 2 -- the push straight from F's CSR entries (path 7), whatever the frontier, in destination slices
  csr0 : the same with push_slices = 0 -- its REDs in entry order
  bits : csr_push = 0 -- the frontier is built as a bit-matrix and the direction-optimising hop runs (push, path 2, below the gate)
  pull : pull_mode = 1 -- the bit-matrix pull (path 3)
  auto : the default dispatch (csr_push.cu: bits_push_from_csr decides between the CSR push and the bit-matrix hop)
Then the same for synthetic hop-2 frontiers whose rows repeat hubs (--synthetic): a pool of vertices of out-degree >= 256 whose
degrees sum to a target `edges`, each of the --sources rows holding each pool vertex with probability ratio / sources, so that
flops / edges is about `ratio`.  Frontiers of more than 2^20 entries (beyond the CSR push's probe) are skipped.
Per frontier it prints hop 2's flops (the mxm flop count), edges (out-degrees summed over the distinct columns of F), the path
each arm took, and the median over --repeats of the hop-2 and hop-2+3 times, CUDA events on the library stream, arms alternated.
The arms' hop-3 results are compared by digest.  Prints one JSON document, with the card's name, power limit and SM clock read in the
same run."""
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


ARMS = {"csr": {"csr_push": 2}, "csr0": {"csr_push": 2, "push_slices": 0}, "bits": {"csr_push": 0}, "pull": {"pull_mode": 1}, "auto": {}}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--sources", type=int, default=512)
    ap.add_argument("--batches", type=int, default=13, help="bench.py's --steps + --warmup")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--synthetic", default="15,30,60:2,3,4,6,10",
                    help="target edges in M : flops/edges ratios of the hub frontiers ('' skips them)")
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("push_gate.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib
    from falkordb_b200.grb import Matrix
    from bench import pick_sources

    fb.init()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    A.prepare(True)
    p, _, _ = A.export_csr()
    deg = np.diff(p.astype(np.int64))
    nnz = int(p[-1])
    batches = pick_sources(deg, a.batches, a.sources, a.seed, 0)
    rows = np.arange(a.sources, dtype=np.uint64)
    strm = torch.cuda.ExternalStream(lib().B200_stream())

    def run_arm(F1, arm):
        """hops 2 and 3 from a copy of the hop-1 CSR; returns (hop-2 ms, hop-2+3 ms, hop-2 path, hop-2 flops, digest)"""
        G = F1.dup()
        fb.sync()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for k, v in ARMS[arm].items():
            fb.set_option(k, v)
        ev[0].record(strm)
        G.lmxm(A)
        ev[1].record(strm)
        path, fl = fb.get_stat("last_path"), fb.get_stat("last_flops")
        for k in ARMS[arm]:
            fb.set_option(k, {"csr_push": 1, "pull_mode": -1, "push_slices": -1}[k])
        G.lmxm(A)
        ev[2].record(strm)
        ev[2].synchronize()
        return ev[0].elapsed_time(ev[1]), ev[0].elapsed_time(ev[2]), int(path), int(fl), G.digest()

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "nnz_A": nnz,
                                        "sources": a.sources, "repeats": a.repeats}, "batches": []}
    print(f"nnz(A) = {nnz}: the edges gate is at {nnz / 4 / 1e6:.1f} M")
    def measure(name, F1, edges):
        t2 = {k: [] for k in ARMS}
        t23 = {k: [] for k in ARMS}
        info = {}
        for r in range(a.repeats + 1):          # the first round is warm-up
            for arm in ARMS:
                ms2, ms23, path, fl, dg = run_arm(F1, arm)
                info[arm] = (path, fl, dg)
                if r:
                    t2[arm].append(ms2)
                    t23[arm].append(ms23)
        flops = {info[k][1] for k in ARMS}
        if len(flops) != 1 or len({tuple(info[k][2]) for k in ARMS}) != 1:
            sys.exit(f"{name}: the arms disagree (flops {flops})")
        row = {"frontier": name, "flops": flops.pop(), "edges": edges, "path": {k: info[k][0] for k in ARMS},
               "hop2_ms": {k: round(statistics.median(v), 3) for k, v in t2.items()},
               "hop23_ms": {k: round(statistics.median(v), 3) for k, v in t23.items()}}
        print(f"{name:>14s} | {row['flops'] / 1e6:7.1f} | {edges / 1e6:7.1f} | {'/'.join(str(row['path'][k]) for k in ARMS)} "
              f"| {' / '.join('%.3f' % row['hop2_ms'][k] for k in ARMS)} | {' / '.join('%.3f' % row['hop23_ms'][k] for k in ARMS)}",
              flush=True)
        return row

    print(f"{'frontier':>14s} | flops M | edges M | path {'/'.join(ARMS)} | hop 2 ms {' / '.join(ARMS)} | hops 2+3 ms {' / '.join(ARMS)}")
    for b, src in enumerate(batches):
        F1 = Matrix(a.sources, n, bool)
        F1.build(rows, src)
        F1.lmxm(A)                              # hop 1, as in the bench
        F1.wait()
        _, fj, _ = F1.export_csr()
        row = measure(f"batch {b}", F1, int(deg[np.unique(fj)].sum()))
        row["batch"] = b
        doc["batches"].append(row)
        del F1
    doc["synthetic"] = []
    if a.synthetic:
        targets, ratios = ([float(x) for x in part.split(",")] for part in a.synthetic.split(":"))
        rng = np.random.default_rng(a.seed)
        cand = rng.permutation(np.nonzero(deg >= 256)[0])
        csum = np.cumsum(deg[cand])
        for te in targets:
            pool = cand[:np.searchsorted(csum, te * 1e6) + 1]
            for ratio in ratios:
                if ratio * len(pool) > (1 << 20):
                    continue
                take = rng.random((a.sources, len(pool))) < ratio / a.sources
                r_, c_ = np.nonzero(take)
                F1 = Matrix(a.sources, n, bool)
                F1.build(r_.astype(np.uint64), pool[c_].astype(np.uint64))
                F1.wait()
                row = measure(f"hubs {te:g}M x{ratio:g}", F1, int(deg[np.unique(pool[c_])].sum()))
                row["target_edges_M"], row["ratio"] = te, ratio
                doc["synthetic"].append(row)
                del F1
    doc["card_after"] = card()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
