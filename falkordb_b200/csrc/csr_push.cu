// csr_push.cu -- Y = F * A pushed straight from a CSR frontier F (in F's entry order, or in L2-sized destination slices), the
// gate that picks it over the bit-matrix hop, and the pending-delta terms of delta_lmxm, which push the deltas' entries.
#include "frontier.cuh"

namespace b200 {

// ---------------------------------------------------------------------------- push straight from a CSR frontier
// Early hops of a traversal batch have a tiny frontier (F in CSR form, a few thousand entries).  Going through the
// bit-matrix there means O(n*W) passes that dwarf the real work (zeroing X, scanning it for flops / active vertices,
// compacting n flags); this path expands F's entries directly: entry (i, k) ORs bit i into Y[j] for every j in A(k,:).
// seen (optional, zeroed, one bit per column of F): *edges += deg(k) over the DISTINCT columns k of F, the edges the bit-matrix
// hop would walk -- the quantity its direction switch compares with nnz(A).
__global__ void k_csr_entry_info(const u64 *__restrict__ Fp, const u32 *__restrict__ Fj, u64 nrows, const u64 *__restrict__ Ap,
                                 u32 *__restrict__ erow, u64 *__restrict__ edeg, u32 *__restrict__ seen, u64 *__restrict__ edges) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u32 lane = threadIdx.x & 31;
    if (warp >= nrows) return;
    u64 ed = 0;
    for (u64 q = Fp[warp] + lane; q < Fp[warp + 1]; q += 32) {
        u32 k = Fj[q];
        erow[q] = (u32)warp;
        const u64 d = Ap[k + 1] - Ap[k];
        edeg[q] = d;
        if (seen) {
            const u32 bit = 1u << (k & 31);
            if (!(atomicOr(seen + (k >> 5), bit) & bit)) ed += d;    // the first entry to claim column k counts its degree
        }
    }
    if (!seen) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ed += __shfl_xor_sync(0xffffffffu, ed, o);
    if (lane == 0 && ed) atomicAdd((unsigned long long *)edges, ed);
}
// One pass over F's entries against the operand's row pointers Ap: erow[q] = the row of entry q, cum[0 .. nnz] = the prefix sums
// of the entries' degrees.  Returns flops = cum[nnz].  edges (optional): also the degrees over F's distinct columns, gathered in
// cum[nnz + 1] (cum then holds nnz + 2 words) and read back with flops in one copy.
static u64 csr_entry_pass(const DevCSR &F, const u64 *Ap, u32 *erow, u64 *cum, u64 *edges) {
    const u64 nnz = F.nnz;
    DevBuf<u32> seen;
    if (edges) {
        seen.alloc((F.ncols + 31) / 32);
        seen.zero();
        CUDA_TRY(cudaMemsetAsync(cum + nnz, 0, 2 * sizeof(u64), stream()));
    }
    LAUNCH(k_csr_entry_info, grid_for(F.nrows * 32, 256), 256, 0, F.p.ptr, F.j.ptr, F.nrows, Ap, erow, cum, seen.ptr,
           edges ? cum + nnz + 1 : nullptr);
    if (!edges) CUDA_TRY(cudaMemsetAsync(cum + nnz, 0, sizeof(u64), stream()));
    exclusive_scan_u64(cum, cum, nnz + 1);
    if (!edges) return read_scalar(cum + nnz);
    u64 h[2];
    d2h(h, cum + nnz, 2);
    sync_stream();
    *edges = h[1];
    return h[0];
}
// ANDNOT (the dirty hop's deleted-edge term, bits_apply_deltas) clears bit i instead of setting it.  SLICED (csr_push_sliced): the
// entries are sub-entries, Ap[e] is where sub-entry e starts in Aj, Fj is not read, and a CTA takes CHUNK flops.
template <int W, bool ANDNOT, bool SLICED = false, u64 CHUNK = PUSH_CHUNK>
__global__ void __launch_bounds__(256)
k_csr_push(const u32 *__restrict__ erow, const u32 *__restrict__ Fj, const u64 *__restrict__ cum, u64 nent, u64 total,
           const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, u64 *__restrict__ Y, const u32 *__restrict__ perm) {
    u64 lo = (u64)blockIdx.x * CHUNK, hi = lo + CHUNK;
    if (hi > total) hi = total;
    for_each_flop(cum, 0, nent, lo, hi, [&](u64 e, u64 t) {
        const u32 i = erow[e];
        u32 col = Aj[(SLICED ? Ap[e] : Ap[Fj[e]]) + (t - cum[e])];
        // hot-set order through the table (the deltas, which have no relabelled copy); a prepared operand passes its
        // relabelled col_idx (PullTables::ap) as Aj instead, with perm null
        if (perm) col = __ldg(perm + col);
        unsigned long long *dst = (unsigned long long *)&Y[(u64)col * W + (i >> 6)];
        if (ANDNOT) atomicAnd(dst, ~(1ULL << (i & 63)));
        else atomicOr(dst, 1ULL << (i & 63));
    });
}
template <int W>
static void csr_push_impl(const DevCSR &F, const DevCSR &A, const u32 *Aj, DevBits &Y, u64 flops, const u32 *erow, const u64 *cum,
                          const u32 *perm, bool acc) {
    u64 nchunks = (flops + PUSH_CHUNK - 1) / PUSH_CHUNK;
    // col_idx + per-entry (row, column, cum) + one RED per flop; the same bytes when accumulating ("bits_push_acc")
    TimedScope ts(acc ? TK_BITS_PUSH_ACC : TK_BITS_PUSH, 4 * flops + 16 * F.nnz + 8 * flops);
    LAUNCH((k_csr_push<W, false>), (u32)nchunks, 256, 0, erow, F.j.ptr, cum, F.nnz, flops, A.p.ptr, Aj, Y.w.ptr, perm);
}
// The same REDs in destination order.  Y is n * W words, many times the L2 on a large graph, and a RED to a record that is not
// resident reads its sector from HBM and writes it back on eviction.  With every row of Aj ascending by position
// (PullTables::ap_sorted), positions [0, n) are cut into P slices of S, and entry (i, k) of F into one sub-entry per slice: the
// part of row k whose positions fall in it, found with one lower bound per (entry, slice boundary).  The non-empty sub-entries
// are listed slice-major -- all of slice 0, then slice 1, ... -- as (row i, first position in Aj, length), and k_csr_push chunks
// the prefix sums of their lengths as it chunks the entries': the flops and the load balance are unchanged, only their order.
// The chunk is SLICE_CHUNK flops, so that the CTAs resident at one time span few slices.
static const u64 SLICE_CHUNK = 512, SLICE_MAX_SUB = (u64)1 << 24, SLICE_MIN_CAP = (u64)1 << 22;
__global__ void k_slice_bounds(const u32 *__restrict__ Fj, u64 nent, const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, u32 P,
                               u64 S, u32 *__restrict__ bnd) {
    const u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nent * (P + 1)) return;
    const u64 e = q / (P + 1), p = q - e * (P + 1);
    const u32 k = Fj[e];
    const u32 *row = Aj + Ap[k];
    u32 lo = 0, hi = (u32)(Ap[k + 1] - Ap[k]);       // the first entry of row k at position >= p * S
    if (p == 0) hi = 0;
    else if (p == P) lo = hi;
    while (lo < hi) {
        const u32 mid = lo + ((hi - lo) >> 1);
        if ((u64)row[mid] < p * S) lo = mid + 1; else hi = mid;
    }
    bnd[q] = lo;
}
// flag[p * nent + e] = sub-entry (e, p) is not empty: slice-major, the order the scan numbers them in
__global__ void k_slice_flags(const u32 *__restrict__ bnd, u64 nent, u32 P, u32 *__restrict__ flag) {
    const u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nent * P) return;
    const u64 p = q / nent, e = q - p * nent;
    flag[q] = bnd[e * (P + 1) + p + 1] > bnd[e * (P + 1) + p];
}
__global__ void k_slice_emit(const u32 *__restrict__ bnd, const u32 *__restrict__ flag, const u64 *__restrict__ pos, u64 nent, u32 P,
                             const u32 *__restrict__ erow, const u32 *__restrict__ Fj, const u64 *__restrict__ Ap,
                             u32 *__restrict__ srow, u64 *__restrict__ sstart, u64 *__restrict__ slen) {
    const u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nent * P || !flag[q]) return;
    const u64 p = q / nent, e = q - p * nent, o = pos[q];
    const u32 b0 = bnd[e * (P + 1) + p];
    srow[o] = erow[e];
    sstart[o] = Ap[Fj[e]] + b0;
    slen[o] = bnd[e * (P + 1) + p + 1] - b0;
}
template <int W>
static void csr_push_sliced(const DevCSR &F, const DevCSR &A, const u32 *Aj, DevBits &Y, u64 flops, const u32 *erow, u32 P, u64 S) {
    const u64 nent = F.nnz, nsub = nent * P;
    // the sub-entry table costs 12 bytes per (entry, boundary) and 20 per non-empty sub-entry, counted at their upper bound
    TimedScope ts(TK_BITS_PUSH, 4 * flops + 16 * F.nnz + 8 * flops + 32 * nsub);
    // One workspace for the six arrays, its capacity a power of two of at least SLICE_MIN_CAP sub-entries: nnz(F) drifts from
    // batch to batch, and a request of a new size class is a cudaMalloc, which costs as much as the push saves, inside the hop.
    u64 cap = SLICE_MIN_CAP;
    while (cap < nsub + nent + 1) cap <<= 1;
    DevBuf<u64> ws(cap * 3 + (cap * 3 + 1) / 2);
    u64 *pos = ws.ptr, *sstart = pos + cap, *scum = sstart + cap;
    u32 *bnd = (u32 *)(scum + cap), *flag = bnd + cap, *srow = flag + cap;
    LAUNCH(k_slice_bounds, grid_for(nent * (P + 1), 256), 256, 0, F.j.ptr, nent, A.p.ptr, Aj, P, S, bnd);
    LAUNCH(k_slice_flags, grid_for(nsub, 256), 256, 0, bnd, nent, P, flag);
    CUDA_TRY(cudaMemsetAsync(flag + nsub, 0, sizeof(u32), stream()));
    exclusive_scan_u32_to_u64(flag, pos, nsub + 1);
    // the slots past the last non-empty sub-entry stay empty: their cum is flops
    CUDA_TRY(cudaMemsetAsync(scum, 0, (nsub + 1) * sizeof(u64), stream()));
    LAUNCH(k_slice_emit, grid_for(nsub, 256), 256, 0, bnd, flag, pos, nent, P, erow, F.j.ptr, A.p.ptr, srow, sstart, scum);
    exclusive_scan_u64(scum, scum, nsub + 1);
    const u64 nchunks = (flops + SLICE_CHUNK - 1) / SLICE_CHUNK;
    LAUNCH((k_csr_push<W, false, true, SLICE_CHUNK>), (u32)nchunks, 256, 0, srow, (const u32 *)nullptr, scum, nsub, flops, sstart, Aj,
           Y.w.ptr, (const u32 *)nullptr);
}
// Whether the push straight from F's CSR entries beats the bit-matrix hop.  edges = the out-degrees summed over the DISTINCT
// columns of F (what the bit-matrix hop walks), flops = over all its entries (one RED each for the CSR push).
//  * edges * 4 > nnz(A): no -- the bit-matrix hop pulls these frontiers.
//  * below that the bit-matrix hop pushes too.  It first spends O(n * W) passes that build, count and compact its frontier (and
//    the next hop packs its natural-order result), then merges the rows that share a column into one RED per word.  So the CSR
//    push wins while its extra REDs, flops - edges, cost less than those passes.  Measured with scripts/push_gate.py on RMAT-24
//    (H100 80GB HBM3, 400 W limit; hops 2 + 3 timed; frontiers of 512 and 1,024 rows that repeat hubs 2 to 14 times): the
//    crossover sits at flops - edges = 0.55, 0.61, 0.70 * n * W at W = 8 and 0.44, 0.48, 0.54 * n * W at W = 16 (edges 15, 30,
//    60 M).  The bound is n * W / 2: it picks the slower route by at most 0.7 ms of the 4 to 22 ms those hops took.  The bench's
//    hop-2 frontiers (W = 8) sit at 0.35 to 0.42.
//  * flops * 4 <= nnz(A) is always taken (it implies the edges bound), as before the bound existed: at W >= 8 that region lies
//    inside the bound; at W = 1 (64 rows: crossover 1.7 to 1.9 * n * W at 15 and 30 M edges, below 2.5 at 60 M) it keeps some
//    frontiers that the bit-matrix hop would take up to 0.4 ms faster.
//  * the sliced push (csr_push_sliced) moved the W = 8 crossover to about 1.0 * n * W where it applies (H100 80GB HBM3, 700 W
//    limit; DESIGN.md 4.8); W = 16 was not re-measured, so the bound stays where no frontier is slower than before it.
static bool csr_push_wins(u64 flops, u64 edges, u64 n, u32 W, u64 nnzA) {
    if (flops * 4 <= nnzA) return true;
    return edges * 4 <= nnzA && (flops - edges) * 2 <= n * W;
}
// Y = F * A from the CSR form of F.  Returns false (nothing done) when the bit-matrix hop should take it (csr_push_wins), unless
// csr_push = 2.  acc: Y |= F * A into a natural-order Y of the product's shape (no zeroing, no vertex order).
bool bits_push_from_csr(const DevCSR &F, const DevCSR &A, DevBits &Y, u64 *flops_out, const PullTables *pt, bool acc) {
    if (F.ncols != A.nrows) throw GrbError(-6, "mxm: inner dimensions differ");
    const u32 W = bits_words_for(F.nrows);
    if (acc) require_acc_target(Y, F.nrows, A.ncols, W);
    u64 flops = 0, edges = 0;
    DevBuf<u32> erow(F.nnz);
    DevBuf<u64> cum(F.nnz + 2);                  // per-entry degrees -> their prefix sums; [nnz] = flops, [nnz + 1] = edges
    if (F.nnz) flops = csr_entry_pass(F, A.p.ptr, erow.ptr, cum.ptr, &edges);
    if (ctx().opt_csr_push != 2 && !csr_push_wins(flops, edges, A.nrows, W, A.nnz)) return false;
    if (!acc) {
        Y.clear();
        Y.nrows = F.nrows; Y.ncols = A.ncols; Y.W = W;
        Y.w.alloc(A.ncols * W);
        Y.w.zero();
    }
    if (flops_out) *flops_out = flops;
    // a square operand with pull tables: write the result in its hot-set order, the form the next pull gathers from directly --
    // through the operand's relabelled col_idx when the tables have it, else through pperm per flop
    const u32 *perm = nullptr, *Aj = A.j.ptr;
    u32 P = 0;                                   // destination slices of the sliced push (0: entry order)
    u64 S = 0;
    if (!acc && pt && ctx().opt_perm_push && pt->perm_tag && pt->pperm && A.nrows == A.ncols && pt->pperm->n == A.ncols) {
        if (pt->ap.ptr && pt->ap.n == A.nnz) Aj = pt->ap.ptr;
        else perm = pt->pperm->ptr;
        // slices of a quarter of the L2, so that the slices the resident CTAs span stay in it together
        const i64 ps = ctx().opt_push_slices;
        if (!perm && pt->ap_sorted && ps != 0 && A.ncols) {
            S = ps > 0 ? (A.ncols + (u64)ps - 1) / (u64)ps : std::max<u64>(1, ctx().l2_bytes / 4 / (8ULL * W));
            const u64 np = (A.ncols + S - 1) / S;
            if ((ps > 0 || np > 1) && np * F.nnz <= SLICE_MAX_SUB) P = (u32)np;
        }
        Y.pvert = pt->pvert;
        Y.pperm = pt->pperm;
        Y.perm_tag = pt->perm_tag;
    }
    if (flops == 0) return true;
    if (P) with_words(W, [&](auto w) { csr_push_sliced<w>(F, A, Aj, Y, flops, erow.ptr, P, S); });
    else with_words(W, [&](auto w) { csr_push_impl<w>(F, A, Aj, Y, flops, erow.ptr, cum.ptr, perm, acc); });
    return true;
}

// ---------------------------------------------------------------------------- pending deltas (delta_lmxm in one pass)
// A dirty hop is F <- (F*m AND NOT F*dm) OR F*dp (matrix.rs:1317-1402, with the reference's over-masking: (i, j) is dropped
// whenever any deleted edge reaches j from row i).  With Y = F*m already computed, the two delta terms need only the deltas'
// entries: for each (k, j) of dm, Y[j] &= ~X[k]; then for each (k, j) of dp, Y[j] |= X[k].  The passes run in stream order,
// every AND-NOT before any OR, which is the phase separation the formula needs.  Work is O(W * nnz(delta)): no pass over the n
// vertices and no product bit-matrix.  X and Y are addressed through the order they are stored in (pperm: vertex ->
// position), so a frontier in hot-set order keeps that order across a dirty hop.
enum { DELTA_ANDNOT = 0, DELTA_OR = 1 };
// delta entries per CTA.  A small delta is spread over n rows, so every entry's row is a binary search over the whole row
// pointer array (about log2(n) dependent loads): short chunks keep that latency chain per CTA short (1 to 8 searches).
static const u64 DELTA_CHUNK = 256;

// The delta's entries in chunks of DELTA_CHUNK per CTA; each entry is handled by SPLIT lanes (the pull's 16-byte record parts),
// which gather their part of X[pos(k)] and reduce it into Y[pos(j)] with RED.AND / RED.OR.  The row k of an entry comes from a
// binary search over the delta's row pointers inside the CTA's row range.  flops += popcount(X[k]) per entry.
template <int W, int OP>
__global__ void __launch_bounds__(256)
k_bits_delta(const u64 *__restrict__ Dp, const u32 *__restrict__ Dj, u64 nrows, u64 nnz, const u64 *__restrict__ X,
             const u32 *__restrict__ xperm, u64 *__restrict__ Y, const u32 *__restrict__ yperm, u64 *__restrict__ flops) {
    constexpr int WL = PullCfg<W>::WL, SPLIT = PullCfg<W>::SPLIT;
    constexpr u32 EPS = 256 / SPLIT;                 // entries per CTA step
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    __shared__ u64 s_r0, s_r1;
    const u64 lo = (u64)blockIdx.x * DELTA_CHUNK;
    const u64 hi = lo + DELTA_CHUNK < nnz ? lo + DELTA_CHUNK : nnz;
    if (threadIdx.x == 0) s_r0 = last_le(Dp, 0, nrows - 1, lo);            // the two bounds are independent searches
    if (threadIdx.x == 32) s_r1 = last_le(Dp, 0, nrows - 1, hi - 1);
    __syncthreads();
    const u64 r1 = s_r1;
    u64 k = s_r0;
    const u32 h = threadIdx.x % SPLIT;
    u64 fl = 0;
    for (u64 q = lo + threadIdx.x / SPLIT; q < hi; q += EPS) {
        k = last_le(Dp, k, r1, q);                   // entries only move forward: the previous row bounds the search
        const u64 j = __ldg(Dj + q);
        const u64 px = xperm ? __ldg(xperm + k) : k, py = yperm ? __ldg(yperm + j) : j;
        u64 x[WL];
        ld_part<WL>(x, X + px * W + h * WL);
        unsigned long long *dst = reinterpret_cast<unsigned long long *>(Y + py * W + h * WL);
#pragma unroll
        for (int w = 0; w < WL; w++) {
            if (!x[w]) continue;
            fl += __popcll(x[w]);
            if (OP == DELTA_OR) atomicOr(dst + w, x[w]);
            else atomicAnd(dst + w, ~x[w]);
        }
    }
    const u64 tot = Red(ts).Sum(fl);
    if (threadIdx.x == 0 && tot) atomicAdd((unsigned long long *)flops, tot);
}

template <int W>
static void bits_delta_impl(const DevBits &X, const DevCSR &D, int op, DevBits &Y, u64 *fl) {
    const u32 *xperm = pos_table(X), *yperm = pos_table(Y);
    const u32 grid = (u32)((D.nnz + DELTA_CHUNK - 1) / DELTA_CHUNK);
    // delta entries (8-byte row pointer share + 4-byte column), the gathered records, the reduced words
    TimedScope ts(TK_BITS_DELTA, 12 * D.nnz + 16ULL * W * D.nnz);
    if (op == DELTA_OR) LAUNCH((k_bits_delta<W, DELTA_OR>), grid, 256, 0, D.p.ptr, D.j.ptr, D.nrows, D.nnz, X.w.ptr, xperm, Y.w.ptr, yperm, fl);
    else LAUNCH((k_bits_delta<W, DELTA_ANDNOT>), grid, 256, 0, D.p.ptr, D.j.ptr, D.nrows, D.nnz, X.w.ptr, xperm, Y.w.ptr, yperm, fl);
}

// The first hop: F is still a CSR of <= 1024 rows and Y came from bits_push_from_csr.  Entry (i, k) of F walks delta row k and
// applies bit i to Y[pos(j)] -- k_csr_push with the delta as its operand, through pperm per flop (a delta has no relabelled
// copy of its col_idx).  Returns flops(F * D).
template <int W>
static u64 csr_delta_impl(const DevCSR &F, const DevCSR &D, int op, DevBits &Y) {
    if (!F.nnz || !D.nnz) return 0;
    DevBuf<u32> erow(F.nnz);
    DevBuf<u64> cum(F.nnz + 1);
    const u64 flops = csr_entry_pass(F, D.p.ptr, erow.ptr, cum.ptr, nullptr);
    if (!flops) return 0;
    const u32 *yperm = pos_table(Y);
    const u32 grid = (u32)((flops + PUSH_CHUNK - 1) / PUSH_CHUNK);
    TimedScope ts(TK_BITS_DELTA, 4 * flops + 16 * F.nnz + 8 * flops);
    if (op == DELTA_OR) LAUNCH((k_csr_push<W, false>), grid, 256, 0, erow.ptr, F.j.ptr, cum.ptr, F.nnz, flops, D.p.ptr, D.j.ptr, Y.w.ptr, yperm);
    else LAUNCH((k_csr_push<W, true>), grid, 256, 0, erow.ptr, F.j.ptr, cum.ptr, F.nnz, flops, D.p.ptr, D.j.ptr, Y.w.ptr, yperm);
    return flops;
}

template <int W>
static u64 apply_deltas_impl(const DevBits *Xb, const DevCSR *Xc, const DevCSR *dm, const DevCSR *dp, DevBits &Y) {
    u64 flops = 0;
    DevBuf<u64> fl;
    const DevCSR *ds[2] = {dm, dp};
    const int ops[2] = {DELTA_ANDNOT, DELTA_OR};
    for (int t = 0; t < 2; t++) {
        const DevCSR *D = ds[t];
        if (!D || !D->nnz) continue;
        if (Xc) { flops += csr_delta_impl<W>(*Xc, *D, ops[t], Y); continue; }
        if (!fl.ptr) { fl.alloc(1); fl.zero(); }
        bits_delta_impl<W>(*Xb, *D, ops[t], Y, fl.ptr);
    }
    if (fl.ptr) flops += read_scalar(fl.ptr);
    return flops;
}

u64 bits_apply_deltas(const DevBits *Xb, const DevCSR *Xc, const DevCSR *dm, const DevCSR *dp, DevBits &Y) {
    const u64 inner = Xc ? Xc->ncols : Xb->ncols;
    for (const DevCSR *D : {dm, dp})
        if (D && (D->nrows != inner || D->ncols != Y.ncols)) throw GrbError(-6, "delta_lmxm: delta dimensions differ from the operand");
    if (!Xc && Xb->W != Y.W) throw GrbError(-101, "delta_lmxm: frontier and product word counts differ");
    require_pos_table(Y, "delta_lmxm");
    if (Xb) require_pos_table(*Xb, "delta_lmxm");
    return with_words(Y.W, [&](auto w) { return apply_deltas_impl<w>(Xb, Xc, dm, dp, Y); });
}

} // namespace b200
