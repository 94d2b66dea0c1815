"""Multi-type hops (-[:R1|R2]->) over relationship types with pending writes: the union hop against the reference's route.

Graph: RMAT-24 (edge factor 16, seed 1) split into T relationship types by a seeded edge hash, for T in --types.  Each type gets
|dp| = |dm| = D for each D in --sizes: dm a seeded random subset of the type's entries, dp seeded random pairs.  Arms, in the same
process, alternated step by step:
  (a) extract : the reference's composition per query -- union_by_extract (extract(T_1), then set_pattern(<!dm_t> m_t) and
                set_pattern(dp_t) per further type, graph.rs:2520-2550) into a fresh matrix, then B200_traverse_batch on it (which
                builds that matrix's transpose mirror and pull tables when a hop pulls)
  (b) union   : B200_traverse_batch_union, every hop a union hop over the types' (m, dp, dm)
  (c) control : B200_traverse_batch over type 1's prepared m alone (one clean type on the same graph)
  (d) no-acc  : (b) with union_accum = 0: a bit-matrix per extra operand, naturalised and ORed in
Workloads: an anchored query (1 source, 1 hop), 512 sources over 1 hop, and 512 sources over a 3-hop chain; a fresh seeded source
batch every step, bitmap hand-off.  A step is one call, timed with CUDA events on the library stream; per row the median over
--steps steps after --warmup.  The outputs of (a), (b) and (d) are compared after every timed step; any difference fails the
script.  Prints one JSON line per row and one JSON document, with the card's name, power limit and SM clock read in the same run."""
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
    ap.add_argument("--types", default="2,3")
    ap.add_argument("--sizes", default="0,256,100000,1000000")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("union_hop.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200._lib import lib
    from falkordb_b200.grb import Descriptor, Matrix

    fb.init()
    n = 1 << a.scale
    A = fb.rmat(a.scale, 16, a.seed)
    p, j, _ = A.export_csr()
    del A
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(p.astype(np.int64)))
    cols = j.astype(np.uint64)
    hsh = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F)) ^ np.uint64(a.seed)) >> np.uint64(61)
    live = np.nonzero(np.diff(p))[0]
    strm = torch.cuda.ExternalStream(lib().B200_stream())
    rng = np.random.default_rng(a.seed)
    wpr = n // 64
    bufs = {k: np.zeros((512, wpr), np.uint64) for k in "abcd"}

    def split(T):
        kind = (hsh % np.uint64(T)).astype(np.int8)
        out = []
        for t in range(T):
            sel = np.nonzero(kind == t)[0]
            pt = np.zeros(n + 1, np.uint64)
            np.cumsum(np.bincount(rows[sel].astype(np.int64), minlength=n), out=pt[1:])
            out.append((Matrix.import_csr(n, n, pt, j[sel], None, bool).prepare(True), sel))
        return out

    def deltas(sel, D):
        dm, dp = Matrix(n, n, bool), Matrix(n, n, bool)
        if D:
            pick = rng.choice(len(sel), size=D, replace=False)
            dm.build(rows[sel][pick], cols[sel][pick])
            dp.build(rng.integers(0, n, D).astype(np.uint64), rng.integers(0, n, D).astype(np.uint64))
        dm.wait(); dp.wait()
        return dp, dm

    def union_by_extract(ops):
        U = Matrix(n, n, bool)
        m, dp, dm = ops[0]
        U.set_pattern(None, m)
        if dm.nvals():
            U.remove_all(dm)
        if dp.nvals():
            U.set_pattern(None, dp)
        for m, dp, dm in ops[1:]:
            U.set_pattern(dm, m, Descriptor.C)
            U.set_pattern(None, dp)
        return U

    def step(arm, src, hops, ops):
        fb.sync()
        out = bufs[arm][:len(src)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(strm)
        if arm == "a":
            U = union_by_extract(ops)
            fb.traverse_batch(src, [U] * hops, fb.OUT_BITMAP, out_bitmap=out)
            del U
        elif arm == "c":
            fb.traverse_batch(src, [ops[0][0]] * hops, fb.OUT_BITMAP, out_bitmap=out)
        else:
            fb.set_option("union_accum", 0 if arm == "d" else 1)
            fb.traverse_batch(src, [[o[0] for o in ops]] * hops, fb.OUT_BITMAP, out_bitmap=out,
                              deltas=[[(o[1], o[2]) for o in ops]] * hops)
            fb.set_option("union_accum", 1)
        e1.record(strm)
        e1.synchronize()
        return e0.elapsed_time(e1)

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}", "steps": a.steps,
                                        "warmup": a.warmup, "hand_off": "bitmap"}, "rows": []}
    for T in [int(s) for s in a.types.split(",")]:
        types = split(T)
        for D in [int(s) for s in a.sizes.split(",")]:
            ops = [(m,) + deltas(sel, D) for m, sel in types]
            for name, nsrc, hops in (("anchored 1 source, 1 hop", 1, 1), ("512 sources, 1 hop", 512, 1), ("512 sources, 3 hops", 512, 3)):
                times = {k: [] for k in "abcd"}
                for s in range(a.warmup + a.steps):
                    src = rng.choice(live, nsrc, replace=False)
                    for arm in "abcd":
                        ms = step(arm, src, hops, ops)
                        if s >= a.warmup:
                            times[arm].append(ms)
                    if s >= a.warmup:
                        k = len(src)
                        if not (np.array_equal(bufs["a"][:k], bufs["b"][:k]) and np.array_equal(bufs["b"][:k], bufs["d"][:k])):
                            sys.exit(f"parity: T = {T}, |delta| = {D}, {name}, step {s}: the union hop differs from the extract route")
                med = {k: round(statistics.median(v), 3) for k, v in times.items()}
                row = {"types": T, "delta_entries_per_type": D, "workload": name, "step_ms": med,
                       "step_ms_min_max": {k: [round(min(v), 3), round(max(v), 3)] for k, v in times.items()},
                       "output_parity_a_b_d": True}
                doc["rows"].append(row)
                print(json.dumps(row), flush=True)
            del ops
        del types
    doc["card_after"] = card()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
