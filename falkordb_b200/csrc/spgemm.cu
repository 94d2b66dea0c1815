// spgemm.cu -- C = pattern(A*B) over GxB_ANY_PAIR_BOOL, row-wise push (Gustavson family).
// Replaces SuiteSparse GB_AxB_saxpy3 as reached from GrB_mxm at
// graph/src/graph/graphblas/matrix.rs:935-943 (lmxm), :956-964 (rmxm), :1346-1394 (delta_lmxm).
//
// Per output row i the work is flops_i = sum_{k in A(i,:)} deg_B(k) column reads.  Rows are binned:
//   flops_i <= small_cap : one CTA stages every B segment of the row in shared memory, bitonic-sorts,
//                          dedupes and writes the sorted run (3 CTA shapes: 64 / 512 / small_cap).
//   flops_i >  small_cap : the row gets an ncols-bit bitmap in global scratch; CTAs each take a
//                          16K-flop chunk of the row (load balanced whatever the degree skew), OR the
//                          bits in with RED.OR, then the bitmap is popcounted, scanned and expanded
//                          straight into the final col_idx array -- already sorted.
// Algorithmic bytes (SURVEY 8d): 4*nnz(A) + 16*nnz(A) [cum/bstart side arrays] + 4*flops + 4*nnz(C).
#include "common.cuh"
#include "ops.cuh"
#include <cub/block/block_scan.cuh>
#include <cub/block/block_reduce.cuh>

namespace b200 {

static const u64 CHUNK_FLOPS = 16384; // flops per CTA in the heavy-row path
static const u32 WB = 1024;           // bitmap words per CTA in count / expand (256 threads x 4)

__global__ void k_entry_deg(const u32 *__restrict__ Aj, u64 nnzA, const u64 *__restrict__ Bp, u64 *__restrict__ w,
                            u64 *__restrict__ bstart) {
    u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; e <= nnzA; e += stride) {
        if (e == nnzA) { w[e] = 0; break; }
        u32 k = Aj[e];
        u64 s = Bp[k], t = Bp[k + 1];
        w[e] = t - s;
        if (bstart) bstart[e] = s;
    }
}

// classes: 0 -> <=64, 1 -> <=512, 2 -> <=cap, 3 -> heavy.  ub[i] = flops for small rows (temp slots).
__global__ void k_classify(const u64 *__restrict__ Ap, const u64 *__restrict__ cum, u64 nrows, u64 cap,
                           u64 *__restrict__ ub, u32 *__restrict__ l0, u32 *__restrict__ l1, u32 *__restrict__ l2,
                           u32 *__restrict__ l3, u32 *__restrict__ counts, u32 *__restrict__ cnt) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i <= nrows; i += stride) {
        if (i == nrows) { ub[i] = 0; break; }
        u64 f = cum[Ap[i + 1]] - cum[Ap[i]];
        u64 u = 0;
        if (f == 0) { cnt[i] = 0; }
        else if (f <= 64) { l0[atomicAdd(&counts[0], 1u)] = (u32)i; u = f; }
        else if (f <= 512) { l1[atomicAdd(&counts[1], 1u)] = (u32)i; u = f; }
        else if (f <= cap) { l2[atomicAdd(&counts[2], 1u)] = (u32)i; u = f; }
        else { l3[atomicAdd(&counts[3], 1u)] = (u32)i; }
        ub[i] = u;
    }
}

template <int CAP, int THREADS>
__global__ void __launch_bounds__(THREADS)
k_small_rows(const u32 *__restrict__ list, u32 nlist, const u64 *__restrict__ Ap, const u64 *__restrict__ cum,
             const u64 *__restrict__ bstart, const u32 *__restrict__ Bj, const u64 *__restrict__ toff,
             u32 *__restrict__ tmp, u32 *__restrict__ cnt) {
    __shared__ u32 buf[CAP];
    typedef cub::BlockScan<u32, THREADS> Scan;
    __shared__ typename Scan::TempStorage ts;
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u32 NW = THREADS / 32;
    for (u32 li = blockIdx.x; li < nlist; li += gridDim.x) {
        u32 row = list[li];
        u64 a0 = Ap[row], a1 = Ap[row + 1];
        u64 base = cum[a0];
        u32 f = (u32)(cum[a1] - base);
        u32 P = 1;
        while (P < f) P <<= 1;
        for (u64 e = a0 + warp; e < a1; e += NW) {
            u64 c0 = cum[e];
            u32 off = (u32)(c0 - base);
            u32 d = (u32)(cum[e + 1] - c0);
            u64 s = bstart[e];
            for (u32 q = lane; q < d; q += 32) buf[off + q] = Bj[s + q];
        }
        for (u32 t = f + tid; t < P; t += THREADS) buf[t] = 0xFFFFFFFFu;
        __syncthreads();
        for (u32 k = 2; k <= P; k <<= 1) {
            for (u32 j = k >> 1; j > 0; j >>= 1) {
                for (u32 t = tid; t < P; t += THREADS) {
                    u32 p = t ^ j;
                    if (p > t) {
                        u32 a = buf[t], b = buf[p];
                        bool up = ((t & k) == 0);
                        if ((a > b) == up) { buf[t] = b; buf[p] = a; }
                    }
                }
                __syncthreads();
            }
        }
        u32 per = (f + THREADS - 1) / THREADS;
        u32 s0 = tid * per, s1 = s0 + per;
        if (s0 > f) s0 = f;
        if (s1 > f) s1 = f;
        u32 local = 0;
        for (u32 t = s0; t < s1; t++) local += (t == 0 || buf[t] != buf[t - 1]) ? 1u : 0u;
        u32 pre, total;
        Scan(ts).ExclusiveSum(local, pre, total);
        u64 o = toff[row] + pre;
        for (u32 t = s0; t < s1; t++)
            if (t == 0 || buf[t] != buf[t - 1]) tmp[o++] = buf[t];
        if (tid == 0) cnt[row] = total;
        __syncthreads();
    }
}

__global__ void k_chunk_counts(const u32 *__restrict__ hrows, u32 nh, const u64 *__restrict__ Ap,
                               const u64 *__restrict__ cum, u64 CH, u64 *__restrict__ nch) {
    u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h > nh) return;
    if (h == nh) { nch[h] = 0; return; }
    u32 row = hrows[h];
    u64 f = cum[Ap[row + 1]] - cum[Ap[row]];
    nch[h] = (f + CH - 1) / CH;
}

// Walks its chunk as common.cuh's for_each_flop does, but in flops counted from the row's first (cum[a0]).  Handing
// for_each_flop the global positions instead changes this kernel's code and takes 4 fewer registers than were measured.
__global__ void __launch_bounds__(256)
k_heavy_accumulate(const u32 *__restrict__ hrows, const u64 *__restrict__ choff, u32 nh, u64 CH,
                   const u64 *__restrict__ Ap, const u64 *__restrict__ cum, const u64 *__restrict__ bstart,
                   const u32 *__restrict__ Bj, u32 *__restrict__ bitmap, u64 wpr) {
    __shared__ u32 s_h;
    __shared__ u64 s_e0, s_e1;
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    u64 c = blockIdx.x;
    if (tid == 0) s_h = (u32)last_le(choff, 0, nh - 1, c);
    __syncthreads();
    u32 h = s_h;
    u32 row = hrows[h];
    u64 lc = c - choff[h];
    u64 a0 = Ap[row], a1 = Ap[row + 1], base = cum[a0], f = cum[a1] - base;
    u64 lo = lc * CH, hi = lo + CH;
    if (hi > f) hi = f;
    if (tid == 0) {
        s_e0 = last_le(cum, a0, a1 - 1, base + lo);
        s_e1 = last_le(cum, a0, a1 - 1, base + hi - 1);
    }
    __syncthreads();
    u64 e0 = s_e0, e1 = s_e1;
    u32 *bm = bitmap + (u64)h * wpr;
    for (u64 t0 = lo + (u64)warp * 32; t0 < hi; t0 += 8 * 32) {
        u64 e = last_le(cum, e0, e1, base + t0);
        u64 t = t0 + lane;
        if (t < hi) {
            while (e < e1 && cum[e + 1] <= base + t) e++;
            u32 col = Bj[bstart[e] + (base + t - cum[e])];
            atomicOr(&bm[col >> 5], 1u << (col & 31));
        }
    }
}

__global__ void __launch_bounds__(256)
k_bitmap_count(const u32 *__restrict__ bitmap, u64 wpr, u32 nb, u64 nblocks, u32 *__restrict__ blkcnt) {
    typedef cub::BlockReduce<u32, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 blk = blockIdx.x;
    if (blk >= nblocks) return;
    u64 h = blk / nb, b = blk % nb;
    const u32 *bm = bitmap + h * wpr;
    u64 w0 = b * WB + (u64)threadIdx.x * 4;
    u32 s = 0;
#pragma unroll
    for (int q = 0; q < 4; q++)
        if (w0 + q < wpr) s += __popc(bm[w0 + q]);
    u32 tot = Red(ts).Sum(s);
    if (threadIdx.x == 0) blkcnt[blk] = tot;
}

__global__ void k_heavy_cnt(const u32 *__restrict__ hrows, u32 nh, u32 nb, const u64 *__restrict__ blkoff,
                            u32 *__restrict__ cnt) {
    u32 h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= nh) return;
    cnt[hrows[h]] = (u32)(blkoff[(u64)(h + 1) * nb] - blkoff[(u64)h * nb]);
}

__global__ void __launch_bounds__(256)
k_bitmap_expand(const u32 *__restrict__ bitmap, u64 wpr, u32 nb, u64 nblocks, const u64 *__restrict__ blkoff,
                const u32 *__restrict__ hrows, const u64 *__restrict__ Cp, u32 *__restrict__ Cj) {
    typedef cub::BlockScan<u32, 256> Scan;
    __shared__ typename Scan::TempStorage ts;
    u64 blk = blockIdx.x;
    if (blk >= nblocks) return;
    u64 h = blk / nb, b = blk % nb;
    const u32 *bm = bitmap + h * wpr;
    u64 w0 = b * WB + (u64)threadIdx.x * 4;
    u32 wd[4];
    u32 s = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        wd[q] = (w0 + q < wpr) ? bm[w0 + q] : 0u;
        s += __popc(wd[q]);
    }
    u32 pre;
    Scan(ts).ExclusiveSum(s, pre);
    u64 o = Cp[hrows[h]] + (blkoff[blk] - blkoff[h * nb]) + pre;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        u32 w = wd[q];
        u32 cbase = (u32)((w0 + q) << 5);
        while (w) {
            u32 bit = __ffs(w) - 1;
            Cj[o++] = cbase + bit;
            w &= w - 1;
        }
    }
}

__global__ void k_gather_small(const u32 *__restrict__ list, u32 nlist, const u64 *__restrict__ toff,
                               const u32 *__restrict__ tmp, const u64 *__restrict__ Cp, u32 *__restrict__ Cj) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 li = warp; li < nlist; li += nwarps) {
        u32 row = list[li];
        u64 s = Cp[row], n = Cp[row + 1] - s, src = toff[row];
        for (u64 q = lane; q < n; q += 32) Cj[s + q] = tmp[src + q];
    }
}

// ---- rows of A with at most one entry: C(i,:) is a copy of one row of B (the first hop of a traversal batch, where
// F(i, src_i) = 1, cond_traverse.rs:600-601).  No sort, no dedupe, no binning: row pointers come straight from the prefix of
// the entry degrees and one warp copies each row.
__global__ void k_single_entry_rows(const u64 *__restrict__ Ap, u64 nrows, u32 *__restrict__ multi) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool b = r < nrows && Ap[r + 1] - Ap[r] > 1;
    if (__any_sync(0xffffffffu, b) && (threadIdx.x & 31) == 0) atomicOr(multi, 1u);
}
__global__ void k_copy_rowptr(const u64 *__restrict__ Ap, u64 nrows, const u64 *__restrict__ cum, u64 *__restrict__ Cp) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r <= nrows) Cp[r] = cum[Ap[r]];          // cum[e] = flops of the entries before e = entries of C before row(e)
}
__global__ void k_copy_rows(const u64 *__restrict__ Ap, u64 nrows, const u64 *__restrict__ cum, const u64 *__restrict__ bstart,
                            const u32 *__restrict__ Bj, u32 *__restrict__ Cj) {
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 r = warp; r < nrows; r += nwarps) {
        u64 e = Ap[r];
        if (Ap[r + 1] == e) continue;
        u64 dst = cum[e], n = cum[e + 1] - dst, src = bstart[e];
        for (u64 q = lane; q < n; q += 32) Cj[dst + q] = Bj[src + q];
    }
}

u64 spgemm_flops(const DevCSR &A, const DevCSR &B) {
    if (A.nnz == 0 || B.nnz == 0) return 0;
    DevBuf<u64> w(A.nnz + 1);
    LAUNCH(k_entry_deg, grid_for(A.nnz + 1, 256, 1 << 16), 256, 0, A.j.ptr, A.nnz, B.p.ptr, w.ptr, (u64 *)nullptr);
    return reduce_sum_u64(w.ptr, A.nnz);
}

void spgemm_anypair(const DevCSR &A, const DevCSR &B, DevCSR &C, u64 *flops_out) {
    Context &cx = ctx();
    if (A.ncols != B.nrows) throw GrbError(-6, "mxm: inner dimensions differ");
    u64 nrows = A.nrows, ncols = B.ncols;
    csr_shape(C, nrows, ncols);
    if (flops_out) *flops_out = 0;
    if (A.nnz == 0 || B.nnz == 0) { C.p.zero(); return; }

    // 1. per-entry degrees, their prefix, and the B segment starts
    DevBuf<u64> cum(A.nnz + 1), bstart(A.nnz);
    LAUNCH(k_entry_deg, grid_for(A.nnz + 1, 256, 1 << 16), 256, 0, A.j.ptr, A.nnz, B.p.ptr, cum.ptr, bstart.ptr);
    exclusive_scan_u64(cum.ptr, cum.ptr, A.nnz + 1);
    DevBuf<u32> multi;
    const bool maybe_single = A.nnz <= nrows;
    if (maybe_single) {
        multi.alloc(1);
        multi.zero();
        LAUNCH(k_single_entry_rows, grid_for(nrows, 256), 256, 0, A.p.ptr, nrows, multi.ptr);
    }
    u64 flops = 0;
    u32 hm = 1;
    d2h(&flops, cum.ptr + A.nnz, 1);
    if (maybe_single) d2h(&hm, multi.ptr, 1);
    sync_stream();                                 // the only host round trip of the single-entry path
    if (flops_out) *flops_out = flops;
    if (flops == 0) { C.p.zero(); return; }
    if (maybe_single) {
        if (!hm) {
            C.nnz = flops;
            C.j.alloc(flops);
            LAUNCH(k_copy_rowptr, grid_for(nrows + 1, 256), 256, 0, A.p.ptr, nrows, cum.ptr, C.p.ptr);
            LAUNCH(k_copy_rows, grid_for(nrows * 32, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, nrows, cum.ptr, bstart.ptr, B.j.ptr, C.j.ptr);
            return;
        }
    }

    // 2. classify rows
    u64 cap = (u64)cx.opt_small_cap;
    if (cap > 4096) cap = 4096;
    if (cap < 512) cap = 512;
    DevBuf<u64> ub(nrows + 1);
    DevBuf<u32> l0(nrows), l1(nrows), l2(nrows), l3(nrows), counts(4), cnt(nrows + 1);
    counts.zero();
    LAUNCH(k_classify, grid_for(nrows + 1, 256, 1 << 16), 256, 0, A.p.ptr, cum.ptr, nrows, cap, ub.ptr, l0.ptr, l1.ptr,
           l2.ptr, l3.ptr, counts.ptr, cnt.ptr);
    u32 hc[4];
    d2h(hc, counts.ptr, 4);
    exclusive_scan_u64(ub.ptr, ub.ptr, nrows + 1); // ub becomes toff
    u64 tmp_total = read_scalar(ub.ptr + nrows);   // also syncs hc
    DevBuf<u32> tmp(tmp_total);

    // 3. small rows
    const u32 maxgrid = (u32)cx.num_sms * 32;
    if (hc[0])
        LAUNCH((k_small_rows<64, 32>), hc[0] < maxgrid * 8 ? hc[0] : maxgrid * 8, 32, 0, l0.ptr, hc[0], A.p.ptr, cum.ptr,
               bstart.ptr, B.j.ptr, ub.ptr, tmp.ptr, cnt.ptr);
    if (hc[1])
        LAUNCH((k_small_rows<512, 64>), hc[1] < maxgrid * 4 ? hc[1] : maxgrid * 4, 64, 0, l1.ptr, hc[1], A.p.ptr, cum.ptr,
               bstart.ptr, B.j.ptr, ub.ptr, tmp.ptr, cnt.ptr);
    if (hc[2])
        LAUNCH((k_small_rows<4096, 256>), hc[2] < maxgrid ? hc[2] : maxgrid, 256, 0, l2.ptr, hc[2], A.p.ptr, cum.ptr,
               bstart.ptr, B.j.ptr, ub.ptr, tmp.ptr, cnt.ptr);

    // 4. heavy rows: bitmap waves
    u32 nh = hc[3];
    u64 wpr = (ncols + 31) / 32;
    u32 nb = (u32)((wpr + WB - 1) / WB);
    u64 budget_rows = (u64)cx.opt_bitmap_budget / (wpr * 4);
    if (budget_rows < 1) budget_rows = 1;
    u64 R = nh < budget_rows ? nh : budget_rows;
    bool single_wave = (nh <= R);
    DevBuf<u32> bitmap, blkcnt;
    DevBuf<u64> blkoff, nch;
    if (nh) {
        bitmap.alloc(R * wpr);
        blkcnt.alloc(R * nb + 1);
        blkoff.alloc(R * nb + 1);
        nch.alloc(R + 1);
    }
    auto accumulate_wave = [&](u32 h0, u32 hn) {
        CUDA_TRY(cudaMemsetAsync(bitmap.ptr, 0, (u64)hn * wpr * 4, stream()));
        LAUNCH(k_chunk_counts, grid_for(hn + 1, 256), 256, 0, l3.ptr + h0, hn, A.p.ptr, cum.ptr, CHUNK_FLOPS, nch.ptr);
        exclusive_scan_u64(nch.ptr, nch.ptr, hn + 1);
        u64 nchunks = read_scalar(nch.ptr + hn);
        if (nchunks > 0x7fffffffULL) throw GrbError(-8, "mxm: too many chunks in one wave");
        {
            TimedScope ts(TK_HEAVY_ACC, 0);
            LAUNCH(k_heavy_accumulate, (u32)nchunks, 256, 0, l3.ptr + h0, nch.ptr, hn, CHUNK_FLOPS, A.p.ptr, cum.ptr,
                   bstart.ptr, B.j.ptr, bitmap.ptr, wpr);
        }
        u64 nblocks = (u64)hn * nb;
        LAUNCH(k_bitmap_count, (u32)nblocks, 256, 0, bitmap.ptr, wpr, nb, nblocks, blkcnt.ptr);
        CUDA_TRY(cudaMemsetAsync(blkcnt.ptr + nblocks, 0, sizeof(u32), stream()));
        exclusive_scan_u32_to_u64(blkcnt.ptr, blkoff.ptr, nblocks + 1);
    };
    for (u32 h0 = 0; h0 < nh; h0 += (u32)R) {
        u32 hn = (nh - h0) < R ? (nh - h0) : (u32)R;
        accumulate_wave(h0, hn);
        LAUNCH(k_heavy_cnt, grid_for(hn, 256), 256, 0, l3.ptr + h0, hn, nb, blkoff.ptr, cnt.ptr);
    }

    // 5. row pointers
    csr_rows_from_counts(cnt.ptr, nrows, C, false);

    // 6. fill
    if (hc[0]) LAUNCH(k_gather_small, grid_for((u64)hc[0] * 32, 256, 1 << 16), 256, 0, l0.ptr, hc[0], ub.ptr, tmp.ptr, C.p.ptr, C.j.ptr);
    if (hc[1]) LAUNCH(k_gather_small, grid_for((u64)hc[1] * 32, 256, 1 << 16), 256, 0, l1.ptr, hc[1], ub.ptr, tmp.ptr, C.p.ptr, C.j.ptr);
    if (hc[2]) LAUNCH(k_gather_small, grid_for((u64)hc[2] * 32, 256, 1 << 16), 256, 0, l2.ptr, hc[2], ub.ptr, tmp.ptr, C.p.ptr, C.j.ptr);
    for (u32 h0 = 0; h0 < nh; h0 += (u32)R) {
        u32 hn = (nh - h0) < R ? (nh - h0) : (u32)R;
        if (!single_wave) accumulate_wave(h0, hn); // bitmap scratch was recycled: rebuild this wave
        u64 nblocks = (u64)hn * nb;
        LAUNCH(k_bitmap_expand, (u32)nblocks, 256, 0, bitmap.ptr, wpr, nb, nblocks, blkoff.ptr, l3.ptr + h0, C.p.ptr, C.j.ptr);
    }
    cx.last_path = 1;
}

} // namespace b200
