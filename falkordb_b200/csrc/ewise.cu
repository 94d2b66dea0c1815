// ewise.cu -- set algebra on sorted CSR rows for the delta-matrix sync half of the path:
//   union      GrB_Matrix_eWiseAdd_BinaryOp  (GxB_ANY_BOOL / GrB_SECOND_UINT64)  matrix.rs:852-874
//   intersect  GrB_Matrix_eWiseMult_Semiring (ANY_PAIR)                           matrix.rs:743-761,876-896
//   filter     mask application / GrB_transpose(...,RCT0) masked copy            matrix.rs:824-845
// (fold formulas versioned_matrix.rs:909-926).  Rows are sorted, so membership / rank of an element in
// the other operand's row is a binary search; output positions are rank sums, which keeps the result
// sorted with no merge loop.  One warp per row, warp-ballot running prefixes inside the row.
// Algorithmic bytes: 4*(nnz(A)+nnz(B)+nnz(C)) + 8*(rows+1)*3 (+8 per valued entry).
#include "common.cuh"
#include "ops.cuh"

namespace b200 {

// ---- predicates -------------------------------------------------------------------------------
struct MaskPred {
    const u64 *Mp; const u32 *Mj; const u64 *Mx; bool comp, structural;
    __device__ bool operator()(u64 i, u32 c, u64) const {
        u64 s = Mp[i], e = Mp[i + 1];
        u64 q = lb32(Mj, s, e, c);
        bool in = (q < e && Mj[q] == c);
        if (in && !structural && Mx) in = (Mx[q] != 0);
        return in != comp;
    }
};
struct RangePred {
    u32 ncols;
    __device__ bool operator()(u64, u32 c, u64) const { return c < ncols; }
};
// keep entry q of the filtered matrix iff its flag bit is set (and, for a valued mask, its own value is non-zero)
struct FlagPred {
    const u32 *flag; const u64 *Mx; bool structural;
    __device__ bool operator()(u64, u32, u64 q) const {
        bool in = (flag[q >> 5] >> (q & 31)) & 1u;
        if (in && !structural && Mx) in = (Mx[q] != 0);
        return in;
    }
};

template <class Pred>
__global__ void k_rowfilter_count(const u64 *__restrict__ Tp, const u32 *__restrict__ Tj, u64 nrows, Pred pred,
                                  u32 *__restrict__ cnt) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 i = warp; i < nrows; i += nwarps) {
        u64 s = Tp[i], e = Tp[i + 1];
        u32 c = 0;
        for (u64 q0 = s; q0 < e; q0 += 32) {
            u64 q = q0 + lane;
            bool keep = (q < e) && pred(i, Tj[q], q);
            c += __popc(__ballot_sync(0xffffffffu, keep));
        }
        if (lane == 0) cnt[i] = c;
    }
}

template <class Pred>
__global__ void k_rowfilter_fill(const u64 *__restrict__ Tp, const u32 *__restrict__ Tj, const u64 *__restrict__ Tx,
                                 u64 nrows, Pred pred, const u64 *__restrict__ Cp, u32 *__restrict__ Cj,
                                 u64 *__restrict__ Cx) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    u32 lt = (1u << lane) - 1u;
    for (u64 i = warp; i < nrows; i += nwarps) {
        u64 s = Tp[i], e = Tp[i + 1];
        u64 o = Cp[i];
        if (Cp[i + 1] == o) continue;
        for (u64 q0 = s; q0 < e; q0 += 32) {
            u64 q = q0 + lane;
            u32 col = (q < e) ? Tj[q] : 0u;
            bool keep = (q < e) && pred(i, col, q);
            u32 m = __ballot_sync(0xffffffffu, keep);
            if (keep) {
                u64 d = o + __popc(m & lt);
                Cj[d] = col;
                if (Cx) Cx[d] = Tx ? Tx[q] : 1ULL;
            }
            o += __popc(m);
        }
    }
}

template <class Pred>
static void rowfilter(const DevCSR &T, Pred pred, u64 out_nrows, u64 out_ncols, bool keep_values, DevCSR &out) {
    csr_shape(out, out_nrows, out_ncols);
    u64 rows = T.nrows < out_nrows ? T.nrows : out_nrows;
    if (T.nnz == 0 || rows == 0) { out.p.zero(); return; }
    DevBuf<u32> cnt(out_nrows + 1);
    timed_begin(TK_FILTER);
    LAUNCH((k_rowfilter_count<Pred>), grid_for(rows * 32, 256, (u64)ctx().num_sms * 32), 256, 0, T.p.ptr, T.j.ptr, rows, pred, cnt.ptr);
    bool vals = keep_values && T.has_values();
    u64 nnz = csr_rows_from_counts(cnt.ptr, rows, out, vals);
    if (nnz)
        LAUNCH((k_rowfilter_fill<Pred>), grid_for(rows * 32, 256, (u64)ctx().num_sms * 32), 256, 0, T.p.ptr, T.j.ptr,
               vals ? T.x.ptr : (const u64 *)nullptr, rows, pred, out.p.ptr, out.j.ptr, vals ? out.x.ptr : (u64 *)nullptr);
    // SURVEY 8(d) bytes_ewise: the operand once, the result once, row pointers of both (+ 8 B per carried value); the probed
    // side (mask / larger operand) is touched by binary searches only and is not counted
    timed_end(TK_FILTER, 4 * (T.nnz + nnz) + 8 * (rows + out_nrows + 2) + (vals ? 8 * (T.nnz + nnz) : 0));
}

void filter_by_mask(const DevCSR &T, const DevCSR &M, bool comp, bool structural, DevCSR &out) {
    if (T.nrows != M.nrows || T.ncols != M.ncols) throw GrbError(-6, "mask dimensions differ");
    MaskPred p{M.p.ptr, M.j.ptr, M.has_values() ? M.x.ptr : nullptr, comp, structural};
    rowfilter(T, p, T.nrows, T.ncols, true, out);
}

void ewise_intersect(const DevCSR &A, const DevCSR &B, DevCSR &out) {
    if (A.nrows != B.nrows || A.ncols != B.ncols) throw GrbError(-6, "eWiseMult dimensions differ");
    // iterate the smaller operand, probe the larger: cost scales with the smaller (versioned_matrix.rs:808-810)
    const DevCSR &S = (A.nnz <= B.nnz) ? A : B;
    const DevCSR &L = (A.nnz <= B.nnz) ? B : A;
    MaskPred p{L.p.ptr, L.j.ptr, nullptr, false, true};
    rowfilter(S, p, A.nrows, A.ncols, false, out);
}

void csr_copy(const DevCSR &A, DevCSR &out, bool keep_values) {
    out.clear();
    out.nrows = A.nrows; out.ncols = A.ncols; out.nnz = A.nnz;
    out.p.alloc(A.nrows + 1);
    d2d(out.p.ptr, A.p.ptr, A.nrows + 1);
    out.j.alloc(A.nnz);
    d2d(out.j.ptr, A.j.ptr, A.nnz);
    if (keep_values && A.has_values()) { out.x.alloc(A.nnz); d2d(out.x.ptr, A.x.ptr, A.nnz); }
}

__global__ void k_extend_rowptr(const u64 *__restrict__ p, u64 old_rows, u64 new_rows, u64 *__restrict__ out) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 last = p[old_rows];
    for (; r <= new_rows; r += stride) out[r] = (r <= old_rows) ? p[r] : last;
}

void csr_resize(const DevCSR &A, u64 nrows, u64 ncols, DevCSR &out) {
    if (nrows >= A.nrows && ncols >= A.ncols) {
        out.clear();
        out.nrows = nrows; out.ncols = ncols; out.nnz = A.nnz;
        out.p.alloc(nrows + 1);
        LAUNCH(k_extend_rowptr, grid_for(nrows + 1, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, A.nrows, nrows, out.p.ptr);
        out.j.alloc(A.nnz);
        d2d(out.j.ptr, A.j.ptr, A.nnz);
        if (A.has_values()) { out.x.alloc(A.nnz); d2d(out.x.ptr, A.x.ptr, A.nnz); }
        return;
    }
    RangePred p{(u32)(ncols > 0xffffffffULL ? 0xffffffffULL : ncols)};
    rowfilter(A, p, nrows, ncols, true, out);
}

// ---- fused masked SpGEMM: Z = pattern(A*B) restricted to the structure of M ---------------------------------------
// C<M> = A*B (ExpandInto-style "which of these candidate pairs are connected through k", BASELINE config 4; also the
// non-complemented mask forms of GrB_mxm).  The output is a subset of M, so nothing outside M is ever materialised: one
// warp per (i,k) entry of A intersects the sorted lists B(k,:) and M(i,:) (the shorter drives, binary search in the
// longer) and sets a flag bit per mask entry; the flagged entries of M are then compacted in order.
// Algorithmic bytes: 4*nnz(A) + 4*flops' + 4*nnz(M) + nnz(M)/8, flops' = sum over (i,k) of min(|B(k,:)|, |M(i,:)|).
__global__ void k_row_ids(const u64 *__restrict__ p, u64 nrows, u32 *__restrict__ rid) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 r = warp; r < nrows; r += nwarps)
        for (u64 q = p[r] + lane; q < p[r + 1]; q += 32) rid[q] = (u32)r;
}
__global__ void __launch_bounds__(256)
k_masked_pairs(const u32 *__restrict__ Arid, const u32 *__restrict__ Aj, u64 nnzA, const u64 *__restrict__ Bp,
               const u32 *__restrict__ Bj, const u64 *__restrict__ Mp, const u32 *__restrict__ Mj, u32 *__restrict__ flag) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 e = warp; e < nnzA; e += nwarps) {
        u32 i = Arid[e], k = Aj[e];
        u64 bs = Bp[k], be = Bp[k + 1], ms = Mp[i], me = Mp[i + 1];
        if (bs == be || ms == me) continue;
        if (be - bs <= me - ms) {                         // B(k,:) drives, probe M(i,:)
            for (u64 q = bs + lane; q < be; q += 32) {
                u32 j = Bj[q];
                u64 pos = lb32(Mj, ms, me, j);
                if (pos < me && Mj[pos] == j) atomicOr(&flag[pos >> 5], 1u << (pos & 31));
            }
        } else {                                          // M(i,:) drives, probe B(k,:); skip already-flagged entries
            for (u64 pz = ms + lane; pz < me; pz += 32) {
                if ((flag[pz >> 5] >> (pz & 31)) & 1u) continue;
                u32 j = Mj[pz];
                u64 pos = lb32(Bj, bs, be, j);
                if (pos < be && Bj[pos] == j) atomicOr(&flag[pz >> 5], 1u << (pz & 31));
            }
        }
    }
}

void spgemm_masked(const DevCSR &A, const DevCSR &B, const DevCSR &M, bool structural, DevCSR &out, u64 flops) {
    if (A.ncols != B.nrows || M.nrows != A.nrows || M.ncols != B.ncols) throw GrbError(-6, "masked mxm: dimension mismatch");
    out.clear();
    out.nrows = M.nrows; out.ncols = M.ncols;
    if (A.nnz == 0 || B.nnz == 0 || M.nnz == 0) { out.p.alloc(M.nrows + 1); out.p.zero(); out.nnz = 0; return; }
    DevBuf<u32> rid(A.nnz), flag((M.nnz + 31) / 32 + 1);
    flag.zero();
    LAUNCH(k_row_ids, grid_for(A.nrows * 32, 256, (u64)ctx().num_sms * 32), 256, 0, A.p.ptr, A.nrows, rid.ptr);
    {
        // SURVEY 8(d) bytes_mxm with the mask term: F's entries and row pointers, A's row-pointer pair per F entry, 4 B per flop (the
        // row-wise bound on the B segments; this kernel reads min(|B(k,:)|, |M(i,:)|) per pair and probes the other side), the mask;
        // the output (a subset of M) is written by the compaction that follows
        TimedScope ts(TK_MASKED, 4 * A.nnz + 4 * (A.nrows + 1) + 8 * A.nnz + 4 * flops + 4 * M.nnz + 4 * (M.nrows + 1));
        LAUNCH(k_masked_pairs, grid_for(A.nnz * 32, 256, (u64)ctx().num_sms * 64), 256, 0, rid.ptr, A.j.ptr, A.nnz, B.p.ptr, B.j.ptr, M.p.ptr,
               M.j.ptr, flag.ptr);
    }
    FlagPred pr{flag.ptr, M.has_values() ? M.x.ptr : nullptr, structural};
    rowfilter(M, pr, M.nrows, M.ncols, false, out);
}

// ---- union ------------------------------------------------------------------------------------
__global__ void k_union_count(const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, const u64 *__restrict__ Bp,
                              const u32 *__restrict__ Bj, u64 nrows, u32 *__restrict__ cnt) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 i = warp; i < nrows; i += nwarps) {
        u64 as = Ap[i], ae = Ap[i + 1], bs = Bp[i], be = Bp[i + 1];
        u32 common = 0;
        if (ae > as && be > bs) {
            // probe the shorter row into the longer one
            bool a_short = (ae - as) <= (be - bs);
            const u32 *Sj = a_short ? Aj : Bj;
            const u32 *Lj = a_short ? Bj : Aj;
            u64 ss = a_short ? as : bs, se = a_short ? ae : be, ls = a_short ? bs : as, le = a_short ? be : ae;
            for (u64 q0 = ss; q0 < se; q0 += 32) {
                u64 q = q0 + lane;
                bool hit = false;
                if (q < se) {
                    u32 c = Sj[q];
                    u64 r = lb32(Lj, ls, le, c);
                    hit = (r < le && Lj[r] == c);
                }
                common += __popc(__ballot_sync(0xffffffffu, hit));
            }
        }
        if (lane == 0) cnt[i] = (u32)((ae - as) + (be - bs) - common);
    }
}

// pos(a_i) = i + lb_B(a_i) - #{common < a_i};   pos(b_j, b_j not in A) = j + lb_A(b_j) - #{common < b_j}
// value on overlap = B's (SECOND, matrix.rs:277-281)
__global__ void k_union_fill(const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, const u64 *__restrict__ Ax,
                             const u64 *__restrict__ Bp, const u32 *__restrict__ Bj, const u64 *__restrict__ Bx,
                             u64 nrows, const u64 *__restrict__ Cp, u32 *__restrict__ Cj, u64 *__restrict__ Cx) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    u32 lt = (1u << lane) - 1u;
    for (u64 i = warp; i < nrows; i += nwarps) {
        u64 as = Ap[i], ae = Ap[i + 1], bs = Bp[i], be = Bp[i + 1];
        u64 o = Cp[i];
        u64 run = 0; // common elements seen so far along a
        for (u64 q0 = as; q0 < ae; q0 += 32) {
            u64 q = q0 + lane;
            bool valid = q < ae, hit = false;
            u32 c = 0;
            u64 r = bs;
            if (valid) {
                c = Aj[q];
                r = lb32(Bj, bs, be, c);
                hit = (r < be && Bj[r] == c);
            }
            u32 m = __ballot_sync(0xffffffffu, hit);
            if (valid) {
                u64 d = o + (q - as) + (r - bs) - (run + __popc(m & lt));
                Cj[d] = c;
                if (Cx) Cx[d] = hit ? (Bx ? Bx[r] : 1ULL) : (Ax ? Ax[q] : 1ULL);
            }
            run += __popc(m);
        }
        run = 0; // common elements seen so far along b
        for (u64 q0 = bs; q0 < be; q0 += 32) {
            u64 q = q0 + lane;
            bool valid = q < be, hit = false;
            u32 c = 0;
            u64 r = as;
            if (valid) {
                c = Bj[q];
                r = lb32(Aj, as, ae, c);
                hit = (r < ae && Aj[r] == c);
            }
            u32 m = __ballot_sync(0xffffffffu, hit);
            if (valid && !hit) {
                u64 d = o + (q - bs) + (r - as) - (run + __popc(m & lt));
                Cj[d] = c;
                if (Cx) Cx[d] = Bx ? Bx[q] : 1ULL;
            }
            run += __popc(m);
        }
    }
}

void ewise_union(const DevCSR &A, const DevCSR &B, bool keep_values, DevCSR &out) {
    if (A.nrows != B.nrows || A.ncols != B.ncols) throw GrbError(-6, "eWiseAdd dimensions differ");
    u64 nrows = A.nrows;
    csr_shape(out, nrows, A.ncols);
    if (nrows == 0 || (A.nnz == 0 && B.nnz == 0)) { out.p.zero(); return; }
    DevBuf<u32> cnt(nrows + 1);
    timed_begin(TK_UNION);
    LAUNCH(k_union_count, grid_for(nrows * 32, 256, (u64)ctx().num_sms * 32), 256, 0, A.p.ptr, A.j.ptr, B.p.ptr, B.j.ptr, nrows, cnt.ptr);
    bool vals = keep_values && (A.has_values() || B.has_values());
    u64 nnz = csr_rows_from_counts(cnt.ptr, nrows, out, vals);
    if (nnz)
        LAUNCH(k_union_fill, grid_for(nrows * 32, 256, (u64)ctx().num_sms * 32), 256, 0, A.p.ptr, A.j.ptr,
               A.has_values() ? A.x.ptr : (const u64 *)nullptr, B.p.ptr, B.j.ptr,
               B.has_values() ? B.x.ptr : (const u64 *)nullptr, nrows, out.p.ptr, out.j.ptr,
               vals ? out.x.ptr : (u64 *)nullptr);
    // SURVEY 8(d) bytes_ewise = 4 * (nnz(A) + nnz(B) + nnz(C)) + row pointers (+ 8 B per valued entry read / written)
    timed_end(TK_UNION, 4 * (A.nnz + B.nnz + nnz) + 8 * 3 * (nrows + 1) + (vals ? 8 * (A.nnz + B.nnz + nnz) : 0));
}


// ---- batched point lookups (ExpandInto) -----------------------------------------------------------------
// found[t] = 1 and val[t] = A(I[t],J[t]) if the entry is stored; one binary search per pair inside the row.
__global__ void k_probe_pairs(const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, const u64 *__restrict__ Ax, u64 nrows,
                              u64 ncols, const u64 *__restrict__ I, const u64 *__restrict__ J, u64 n,
                              unsigned char *__restrict__ found, u64 *__restrict__ val) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        u64 i = I[t], j = J[t];
        bool hit = false;
        u64 v = 0;
        if (i < nrows && j < ncols) {
            u64 s = Ap[i], e = Ap[i + 1];
            u64 q = lb32(Aj, s, e, (u32)j);
            if (q < e && Aj[q] == (u32)j) { hit = true; v = Ax ? Ax[q] : 1ULL; }
        }
        found[t] = hit ? 1 : 0;
        if (val) val[t] = v;
    }
}
void probe_pairs(const DevCSR &A, const u64 *dI, const u64 *dJ, u64 n, unsigned char *d_found, u64 *d_val) {
    if (n) LAUNCH(k_probe_pairs, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, A.j.ptr, A.has_values() ? A.x.ptr : (const u64 *)nullptr,
                  A.nrows, A.ncols, dI, dJ, n, d_found, d_val);
}

// ---- hypersparse host form <-> dense device rowptr ---------------------------------------------
// p[r] = hptr[ first vector index with hrow >= r ]  (hrow ascending, nvec entries, hptr[nvec] = nnz)
__global__ void k_rowptr_from_hyper(const u64 *__restrict__ hrow, const u64 *__restrict__ hptr, u64 nvec, u64 nrows,
                                    u64 *__restrict__ p) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; r <= nrows; r += stride) p[r] = hptr[lb64(hrow, 0, nvec, r)];
}
void rowptr_from_hyper(const u64 *d_hrow, const u64 *d_hptr, u64 nvec, u64 nrows, u64 *d_p) {
    LAUNCH(k_rowptr_from_hyper, grid_for(nrows + 1, 256, (u64)ctx().num_sms * 16), 256, 0, d_hrow, d_hptr, nvec, nrows, d_p);
}

__global__ void k_flag_nonempty(const u64 *__restrict__ p, u64 nrows, u32 *__restrict__ flag) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; r <= nrows; r += stride) flag[r] = (r < nrows && p[r + 1] > p[r]) ? 1u : 0u;
}
__global__ void k_scatter_hyper(const u64 *__restrict__ p, const u32 *__restrict__ flag, const u64 *__restrict__ pos,
                                u64 nrows, u64 *__restrict__ hrow, u64 *__restrict__ hptr) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; r < nrows; r += stride)
        if (flag[r]) { hrow[pos[r]] = r; hptr[pos[r]] = p[r]; }
}
// returns nvec; d_hrow / d_hptr (nvec+1, last = nnz) are allocated here
u64 hyper_from_rowptr(const u64 *d_p, u64 nrows, u64 nnz, DevBuf<u64> &d_hrow, DevBuf<u64> &d_hptr) {
    DevBuf<u32> flag(nrows + 1);
    DevBuf<u64> pos(nrows + 1);
    LAUNCH(k_flag_nonempty, grid_for(nrows + 1, 256, (u64)ctx().num_sms * 16), 256, 0, d_p, nrows, flag.ptr);
    exclusive_scan_u32_to_u64(flag.ptr, pos.ptr, nrows + 1);
    u64 nvec = read_scalar(pos.ptr + nrows);
    d_hrow.alloc(nvec ? nvec : 1);
    d_hptr.alloc(nvec + 1);
    if (nvec) LAUNCH(k_scatter_hyper, grid_for(nrows, 256, (u64)ctx().num_sms * 16), 256, 0, d_p, flag.ptr, pos.ptr, nrows, d_hrow.ptr, d_hptr.ptr);
    fill_u64(d_hptr.ptr + nvec, nnz, 1);
    return nvec;
}


// ---- order-sensitive digest of a CSR pattern (full-size parity checks: a multi-GB result is compared by three numbers) ----
// key = row << 32 | col, position q = index in CSR order:  d[0] = nnz, d[1] = sum mix(key), d[2] = sum mix(key + GOLD * (q + 1)).
// Same arithmetic as oracle/grb_oracle.c: orc_digest (the CPU side hashes the oracle's result).
__device__ __forceinline__ u64 mix64(u64 x) {
    x ^= x >> 33; x *= 0xFF51AFD7ED558CCDULL; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ULL; x ^= x >> 33;
    return x;
}
__global__ void __launch_bounds__(256) k_csr_digest(const u64 *__restrict__ p, const u32 *__restrict__ j, u64 nrows, u64 nnz, u64 *__restrict__ d) {
    u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    u64 s1 = 0, s2 = 0;
    u64 row = 0;                                   // rows only move forward along a thread's ascending positions
    for (; q < nnz; q += stride) {
        if (p[row + 1] <= q) row = last_le(p, row + 1, nrows - 1, q);   // largest row with p[row] <= q, searched in (row, nrows)
        const u64 key = (row << 32) | j[q];
        s1 += mix64(key);
        s2 += mix64(key + 0x9E3779B97F4A7C15ULL * (q + 1));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
    if ((threadIdx.x & 31) == 0) { atomicAdd((unsigned long long *)&d[1], s1); atomicAdd((unsigned long long *)&d[2], s2); }
}
void csr_digest(const DevCSR &A, u64 *host_out3) {
    DevBuf<u64> d(3);
    d.zero();
    if (A.nnz) LAUNCH(k_csr_digest, grid_for(A.nnz, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, A.j.ptr, A.nrows, A.nnz, d.ptr);
    u64 h[3] = {0, 0, 0};
    d2h(h, d.ptr, 3);
    sync_stream();
    host_out3[0] = A.nnz; host_out3[1] = h[1]; host_out3[2] = h[2];
}

} // namespace b200
