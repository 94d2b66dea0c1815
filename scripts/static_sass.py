#!/usr/bin/env python
"""Static evidence for kernels that have no ncu capture: registers / shared memory / spills (cuobjdump -res-usage) and the memory
instruction mix of the SASS (cuobjdump -sass) of the shipped libb200grb.so, for the instantiations the default options launch.
Needs no GPU.  Usage: python scripts/static_sass.py > static_sass.md"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "falkordb_b200", "libb200grb.so")
# demangled-name prefixes of the instantiations the 512-source chain (W = 8), the BFS engine and the side kernels launch
WANT = [
    ("hop, pull (mid + long-row segments), W = 8, L2 policies", r"k_pull_seg<8, true, 4, false, false>"),
    ("hop, pull (rows <= 8), W = 8, L2 policies", r"k_pull_small<8, true, false>"),
    ("hop 2, CSR push", r"k_csr_push<8"),
    ("frontier totals in gather order", r"k_ordered_flops<8>"),
    ("materialise, count (carry-save)", r"k_bits_count_csa<8>"),
    ("materialise, fill", r"k_bits_fill<8>"),
    ("bitmap hand-off", r"k_bits_rowmajor"),
    ("BFS top-down expand", r"k_do_expand<false>"),
    ("BFS bottom-up", r"k_do_pull<false>"),
    ("BFS parent assign", r"k_do_assign<false>"),
    ("BFS top-down expand, operands with deltas", r"k_do_expand<true>"),
    ("BFS bottom-up, operands with deltas", r"k_do_pull<true>"),
    ("BFS parent assign, operands with deltas", r"k_do_assign<true>"),
    ("masked SpGEMM pairs", r"k_masked_pairs"),
    ("set union", r"k_union"),
    ("mask filter", r"k_rowfilter_fill"),
    ("adjacency layer, count (identity form)", r"k_adj_layer<b200::RankIdentity, false>"),
    ("adjacency layer, fill (identity form)", r"k_adj_layer<b200::RankIdentity, true>"),
    ("adjacency layer, count (kept list)", r"k_adj_layer<b200::RankTable, false>"),
    ("adjacency layer, fill (kept list)", r"k_adj_layer<b200::RankTable, true>"),
    ("FP64 mxv (PLUS_SECOND)", r"k_mxv_fp64<false>"),
    ("WCC hook", r"k_cc_hook"),
    ("CDLP pick", r"k_cdlp_pick"),
    ("bulk tensor build, run marking", r"k_bulk_mark"),
    ("relationship ids, count", r"k_ee_count"),
    ("relationship ids, fill", r"k_ee_fill"),
    ("insert plan, count", r"k_ins_count"),
    ("insert plan, fill", r"k_ins_fill"),
    ("remove plan, count", r"k_rm_count"),
    ("remove plan, fill", r"k_rm_fill"),
    ("sorted keys, run heads", r"k_run_heads"),
    ("relationship ids, reference order fill", r"k_ee_ref_fill"),
    ("trails, candidates", r"k_tr_cand"),
    ("trails, stored level fill", r"k_tr_fill"),
    ("trails, last-level emissions", r"k_tr_out_last"),
    ("trails, stored-level emissions", r"k_tr_out("),
    ("bidirectional reach, closure hits", r"k_vb_hit"),
    ("bidirectional reach, closure row mask", r"k_vb_mask"),
    ("bidirectional reach, closure seeds", r"k_vb_seed("),
    ("bidirectional reach, start fix-up (CSR)", r"k_vb_fix_copy"),
    ("shortest path, neighbour emission", r"k_sp_emit"),
    ("shortest path, distinct entries and meets", r"k_sp_classify"),
    ("shortest path, path write", r"k_sp_write"),
]
OPS = [("LDG.*\\.256", r"\bLDG\.[A-Z0-9_.]*256"), ("LDG.*\\.128", r"\bLDG\.[A-Z0-9_.]*128"), ("LDG.*\\.64", r"\bLDG\.[A-Z0-9_.]*\.64\b"),
       ("LDG other", r"\bLDG\."), ("STG.*\\.256", r"\bSTG\.[A-Z0-9_.]*256"), ("STG.*\\.128", r"\bSTG\.[A-Z0-9_.]*128"), ("STG other", r"\bSTG\."),
       ("REDG (global reduction)", r"\bREDG\."), ("ATOMG", r"\bATOMG\."), ("ATOMS", r"\bATOMS\."), ("REDUX", r"\bREDUX\b"), ("LDS/STS", r"\b(LDS|STS)\b"), ("SHFL", r"\bSHFL\."), ("VOTE/MATCH", r"\b(VOTE|MATCH)\b"),
       ("POPC", r"\bPOPC\b"), ("PRMT", r"\bPRMT\b"), ("LOP3", r"\bLOP3\b"), ("BAR", r"\bBAR\.")]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    res = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True).stdout
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            usage[cur] = dict(re.findall(r"(REG|STACK|SHARED|LOCAL):(\d+)", line))
            cur = None
    dm = demangle(list(usage))
    sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True).stdout
    bodies, cur = collections.defaultdict(list), None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and re.match(r"\s*/\*[0-9a-f]{4}\*/", line):
            bodies[cur].append(line)
    print("# Static SASS evidence (no GPU needed): `python scripts/static_sass.py` on the shipped `libb200grb.so` (sm_90a)\n")
    print("Registers / shared memory / spills per thread block and the memory-instruction mix of the instantiations the default options launch.")
    print("`LDG.*.128` / `STG.*.128` are the widest (16-byte) global accesses on sm_90; `REDG` = fire-and-forget global atomics (OR / ADD / MIN).\n")
    print("| kernel | instantiation | regs | smem B | spill B | SASS lines | " + " | ".join(n for n, _ in OPS) + " |")
    print("|---|---|---|---|---|---|" + "---|" * len(OPS))
    for label, pat in WANT:
        hits = [k for k, v in dm.items() if pat in v]
        if not hits:
            print(f"| {label} | `{pat}` not found | | | | |" + " |" * len(OPS))
            continue
        k = sorted(hits, key=lambda x: len(dm[x]))[0]
        u = usage[k]
        body = bodies.get(k, [])
        counts, seen = [], set()
        for name, rx in OPS:
            c = 0
            for i, ln in enumerate(body):
                if i in seen:
                    continue
                if re.search(rx, ln):
                    c += 1
                    seen.add(i)
            counts.append(c)
        short = dm[k].split("(")[0].replace("void b200::", "").replace("b200::", "")
        print(f"| {label} | `{short}` | {u.get('REG')} | {u.get('SHARED')} | {u.get('LOCAL')} | {len(body)} | " + " | ".join(str(c) for c in counts) + " |")
    spills = [dm[k] for k, u in usage.items() if int(u.get("LOCAL", 0)) > 0]
    print(f"\nKernels in the library: {len(usage)}; with local-memory spills: {len(spills)}" + (": " + "; ".join(s.split('(')[0] for s in spills[:8]) if spills else "") + ".")


if __name__ == "__main__":
    sys.exit(main())
