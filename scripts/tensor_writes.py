"""Relationship inserts and deletes: Tensor::set_all_from_slices / remove_all with the read phase on the host (the reference route)
against set_all_from_slices_dev / remove_all_dev, whose read phase is one B200_Tensor_insert_plan / B200_Tensor_remove_plan call.

Graph: RMAT-24 (edge factor 16, seed 1) with edge ids in COO order, plus a share (--multi) of pairs carrying a second edge (new
ids), split into T relationship types by a seeded edge hash, for T in --types.  Each type is loaded twice by Tensor::bulk_load
(base built on the device, no host form): one twin is written through the reference route, the other through the device route.
  cold : one single-edge insert per type on fresh twins.  The reference route's first probe downloads the type's base m and its
         transpose mt (GrB_Matrix_extractElement on a base without host form); the device route's does not.
  grid : per batch size b in --batches, an insert batch (3/4 random pairs, 1/4 pairs already loaded: promotions; fresh ids) and a
         delete batch (half the ids on multi-edge pairs, half on single-edge pairs; loaded edges not deleted before) on every type,
         reference route (warm) then device route.
After every call the twins are compared: digests of m and mt's base, every entry of the seven other layers, the six Delta
counters, edge_count, and the emptied pairs of deletes; any difference fails the script.  A call is timed on the host clock (it
ends in host-side writes after a device synchronise).  d2h_bytes is the library's device-to-host byte count over the call.
tensor_write GB/s is the plan kernels' compulsory bytes (writes.cu) over their CUDA-event time, with its fraction of 3.35 TB/s.
Prints one JSON line per row and one JSON document, with the card's name, power limit and SM clock read in the same run."""
import argparse
import ctypes as C
import json
import os
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


def state(t):
    """what the twins must agree on: digests of m and mt's base, the other seven layers' entries, counters, edge_count"""
    import falkordb_b200 as fb
    from falkordb_b200 import host_mirror as hm
    hs = t.layers()
    out = []
    for k, h in enumerate(hs):
        if k in (0, 3):
            d = np.zeros(3, np.uint64)
            fb.check(fb.lib().B200_Matrix_digest(C.c_void_p(h), d.ctypes.data))
            out.append(d)
        else:
            out.extend(x for x in hm._tuples(h, k < 2) if x is not None)
    out.append(t.counts())
    out.append(np.array([t.edge_count()], np.uint64))
    return out


def same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(state(a), state(b)))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--types", default="1,3")
    ap.add_argument("--batches", default="1,1000,100000,1000000")
    ap.add_argument("--multi", type=float, default=0.01, help="share of pairs that get a second edge")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--out", default=None, help="also write the JSON document here")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        sys.exit("tensor_writes.py measures on the GPU: no CUDA device")
    import falkordb_b200 as fb
    from falkordb_b200 import host_mirror as hm
    from falkordb_b200._lib import lib

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
    is_multi = np.zeros(len(cols) + len(extra), bool)
    is_multi[extra] = True
    is_multi[len(cols):] = True
    rows = np.concatenate([rows, rows[extra]])
    cols = np.concatenate([cols, cols[extra]])
    ids = np.concatenate([ids, np.arange(len(ids), len(ids) + len(extra), dtype=np.uint64)])
    hsh = ((rows * np.uint64(0x9E3779B97F4A7C15)) ^ (cols * np.uint64(0xC2B2AE3D27D4EB4F)) ^ np.uint64(a.seed)) >> np.uint64(61)
    batches = [int(s) for s in a.batches.split(",")]

    def timed(f):
        lib().B200_reset_stats()
        t0 = time.perf_counter()
        out = f()
        ms = (time.perf_counter() - t0) * 1e3
        return ms, int(fb.get_stat("d2h_bytes")), out

    def kernel():
        ms, nl, by = C.c_double(0), C.c_uint64(0), C.c_uint64(0)
        lib().B200_kernel_stats(b"tensor_write", C.byref(ms), C.byref(nl), C.byref(by))
        return ms.value, by.value

    doc = {"card": card(), "workload": {"graph": f"RMAT-{a.scale}, edge factor 16, seed {a.seed}, ids in COO order, "
                                                 f"{a.multi:.0%} of pairs with a second edge", "batches": batches,
                                        "timing": "host clock around each call, one call per arm"},
           "rows": []}
    next_id = len(ids)
    for T in [int(s) for s in a.types.split(",")]:
        kind = (hsh % np.uint64(T)).astype(np.int8)
        twins, pools = [], []
        for t in range(T):
            sel = np.nonzero(kind == t)[0]
            twins.append((hm.Tensor(n, rows[sel], cols[sel], ids[sel]), hm.Tensor(n, rows[sel], cols[sel], ids[sel])))
            order = rng.permutation(sel)                            # deletes draw from here, each edge once
            pools.append({"multi": list(order[is_multi[order]]), "single": list(order[~is_multi[order]]), "sel": sel})

        def run(op, b, t, cold=False):
            ref, dev = twins[t]
            if op == "insert":
                q = b - b // 4
                old = rng.choice(pools[t]["sel"], b // 4)
                ns = np.concatenate([rng.integers(0, n, q).astype(np.uint64), rows[old]])
                nd = np.concatenate([rng.integers(0, n, q).astype(np.uint64), cols[old]])
                nid = np.arange(next_id, next_id + b, dtype=np.uint64)
                f_ref = lambda: ref.add(ns, nd, nid, route=hm.WRITE_REFERENCE)
                f_dev = lambda: dev.add(ns, nd, nid, route=hm.WRITE_DEVICE)
            else:
                hm_, hs_ = b // 2, b - b // 2
                take = pools[t]["multi"][:hm_] + pools[t]["single"][:hs_]
                del pools[t]["multi"][:hm_], pools[t]["single"][:hs_]
                g = np.array(take, np.int64)
                f_ref = lambda: ref.remove(ids[g], rows[g], cols[g], route=hm.WRITE_REFERENCE)
                f_dev = lambda: dev.remove(ids[g], rows[g], cols[g], route=hm.WRITE_DEVICE)
            ms_r, d2h_r, e_r = timed(f_ref)
            fb.set_option("timing", 1)
            ms_d, d2h_d, e_d = timed(f_dev)
            kms, kby = kernel()
            fb.set_option("timing", 0)
            if op == "delete" and set(map(tuple, e_r.tolist())) != set(map(tuple, e_d.tolist())):
                sys.exit(f"parity: emptied pairs differ ({T} types, type {t}, {op} {b})")
            if not same(ref, dev):
                sys.exit(f"parity: the twins differ ({T} types, type {t}, {op} {b})")
            return {"types": T, "type": t, "op": op, "batch": b, "reference": "cold" if cold else "warm",
                    "ms": {"reference": round(ms_r, 3), "device": round(ms_d, 3)},
                    "speedup": round(ms_r / ms_d, 2) if ms_d else None, "d2h_bytes": {"reference": d2h_r, "device": d2h_d},
                    "tensor_write_kernel_ms": round(kms, 4), "tensor_write_bytes": kby,
                    "tensor_write_GBps": round(kby / kms / 1e6, 1) if kms else None,
                    "tensor_write_frac_of_3_35TBps": round(kby / kms / 1e6 / HBM_GBS, 4) if kms else None, "parity": True}

        for t in range(T):
            row = run("insert", 1, t, cold=True)
            next_id += 1
            doc["rows"].append(row)
            print(json.dumps(row), flush=True)
        for b in batches:
            for op in ("insert", "delete"):
                for t in range(T):
                    row = run(op, b, t)
                    if op == "insert":
                        next_id += b
                    doc["rows"].append(row)
                    print(json.dumps(row), flush=True)
        del twins
    doc["card_after"] = card()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()
