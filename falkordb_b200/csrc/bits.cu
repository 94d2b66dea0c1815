// bits.cu -- frontier bit-matrix path.
//
// FalkorDB's CondTraverse drives GrB_mxm with a short-fat left operand: F is |batch| x n with
// |batch| <= 1024 rows (graph/src/runtime/batch.rs:81, runtime/ops/cond_traverse.rs:600-605).
// For such operands the row-wise product F*A is the multi-source frontier expansion
//        Y[j] |= X[k]   for every edge (k,j) of A,    X[k] = bitmask of the F rows holding k,
// i.e. ONE pass over A serves up to 64*W frontier rows at once.  F lives as a vertex-major
// bit-matrix (DevBits) between hops; the sorted CSR the reference iterates
// (matrix.rs:1471-1605) is materialised only when something observes it.
//   push : active vertices only, load-balanced flat expansion, RED.OR.64 into Y
//   pull : stream A' (CSC of A) row by row, gather X[k], plain stores -- no atomics
// Algorithmic bytes per hop (pull): 4*nnz(A') + 8*(n+1) + 8*W*nnz(A') gathers (L2) + 8*W*n.
#include "common.cuh"
#include "ops.cuh"
#include <cub/block/block_reduce.cuh>

namespace b200 {

// how the lanes of a warp share a W-word vertex record: a lane moves at most 16 bytes per instruction on sm_90 (LDG.128 / STG.128)
__host__ __device__ constexpr int pull_split(int W) { return W >= 2 ? W / 2 : 1; }
template <int W> struct PullCfg {
    static constexpr int SPLIT = pull_split(W);    // lanes per vertex record
    static constexpr int WL = W / SPLIT;           // words per lane
    static constexpr int VG = 8 / SPLIT;           // vertices gathered per 8-lane group and unroll step
};
static const u64 PUSH_CHUNK = 8192;
static const u64 LONG_ROW = 4096;   // pull: rows longer than this are split into LONG_ROW-entry segments

static void require_natural(const DevBits &X, const char *what);
// accumulate mode (union hops): the product is ORed into Y, which must already hold a natural-order product of the same shape
static void require_acc_target(const DevBits &Y, u64 nrows, u64 ncols, u32 W) {
    require_natural(Y, "accumulating product");
    if (Y.nrows != nrows || Y.ncols != ncols || Y.W != W) throw GrbError(-6, "accumulating product: target shape differs");
}

u32 bits_words_for(u64 nrows) {
    if (nrows == 0) return 1;
    u64 w = (nrows + 63) / 64;
    if (w > 16) return 0;
    u32 p = 1;
    while (p < w) p <<= 1;
    return p;
}

// ---------------------------------------------------------------------------- CSR -> bits
__global__ void k_bits_scatter(const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, u64 nrows, u64 nnz,
                               u64 *__restrict__ X, u32 W) {
    u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; q < nnz; q += stride) {
        // row = largest r with Ap[r] <= q
        u64 lo = 0, hi = nrows - 1;
        while (lo < hi) {
            u64 mid = (lo + hi + 1) >> 1;
            if (Ap[mid] <= q) lo = mid; else hi = mid - 1;
        }
        u32 col = Aj[q];
        atomicOr((unsigned long long *)&X[(u64)col * W + (lo >> 6)], 1ULL << (lo & 63));
    }
}

void bits_from_csr(const DevCSR &F, DevBits &X) {
    u32 W = bits_words_for(F.nrows);
    if (!W) throw GrbError(-8, "bit-frontier form needs <= 1024 rows");
    X.clear();
    X.nrows = F.nrows; X.ncols = F.ncols; X.W = W;
    X.w.alloc(F.ncols * W);
    X.w.zero();
    if (F.nnz)
        LAUNCH(k_bits_scatter, grid_for(F.nnz, 256, 1 << 16), 256, 0, F.p.ptr, F.j.ptr, F.nrows, F.nnz, X.w.ptr, W);
}

// ---------------------------------------------------------------------------- bits -> CSR
// Materialise the sorted CSR the reference's row iterator walks (matrix.rs:1471-1605) from the vertex-major
// bit-matrix.  A warp owns 32 consecutive vertices; a 5-stage shuffle butterfly transposes their 32x32 bit
// block so lane b holds "which of my 32 vertices are in frontier row b" (and row 32+b for the high half).
// Count pass: popcounts per (tile, row), laid out row-major-by-tile so ONE global exclusive scan yields final
// CSR positions.  Fill pass: a warp expands one row's masks into a shared-memory list (u16 tile-local ids),
// then the row segment is copied out with coalesced stores -- ascending vertex id within each row.
static const u32 TILE_V = 1024;          // vertices per CTA tile
static const u32 TILE_THREADS = 512;     // 16 warps x 2 groups of 32 vertices

__device__ __forceinline__ u32 transpose32(u32 x, u32 lane) {
    // bit c of lane l  ->  bit l of lane c
    u32 y;
    y = __shfl_xor_sync(0xffffffffu, x, 16);
    x = (lane & 16) ? ((x & 0xFFFF0000u) | ((y & 0xFFFF0000u) >> 16)) : ((x & 0x0000FFFFu) | ((y & 0x0000FFFFu) << 16));
    y = __shfl_xor_sync(0xffffffffu, x, 8);
    x = (lane & 8) ? ((x & 0xFF00FF00u) | ((y & 0xFF00FF00u) >> 8)) : ((x & 0x00FF00FFu) | ((y & 0x00FF00FFu) << 8));
    y = __shfl_xor_sync(0xffffffffu, x, 4);
    x = (lane & 4) ? ((x & 0xF0F0F0F0u) | ((y & 0xF0F0F0F0u) >> 4)) : ((x & 0x0F0F0F0Fu) | ((y & 0x0F0F0F0Fu) << 4));
    y = __shfl_xor_sync(0xffffffffu, x, 2);
    x = (lane & 2) ? ((x & 0xCCCCCCCCu) | ((y & 0xCCCCCCCCu) >> 2)) : ((x & 0x33333333u) | ((y & 0x33333333u) << 2));
    y = __shfl_xor_sync(0xffffffffu, x, 1);
    x = (lane & 1) ? ((x & 0xAAAAAAAAu) | ((y & 0xAAAAAAAAu) >> 1)) : ((x & 0x55555555u) | ((y & 0x55555555u) << 1));
    return x;
}

// Count pass with vertical counters.  The counts per (frontier row, tile) are a positional
// popcount: for each of the 64 bit positions of a word column, how many of the tile's 1024 words have that bit set.  No bit
// transpose per 32 vertices is needed for that: a lane adds the words of 32 vertices (v = lane, lane + 32, ...) into a
// carry-save adder tree -- 31 CSAs of two LOP3 per 32-bit half leave six bit-planes (weights 1, 2, .., 32) -- and only the
// planes are transposed across the warp (12 butterflies per word column instead of 64): ~4x fewer instructions than
// transposing every word.  One warp per (tile, group of up to 4 word columns); loads are 8*WL contiguous bytes per lane.
__device__ __forceinline__ void csa(u64 &hi, u64 &lo, u64 a, u64 b, u64 c) {   // a + b + c = 2 * hi + lo, bitwise
    const u64 u = a ^ b;
    hi = (a & b) | (u & c);
    lo = u ^ c;
}
template <int WL> __device__ __forceinline__ void ld_part(u64 (&x)[WL], const u64 *p) {
    static_assert(WL == 1 || WL == 2, "a record part is one 8- or 16-byte load");
    if constexpr (WL == 1) { x[0] = __ldg(p); }
    else { ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(p)); x[0] = v.x; x[1] = v.y; }
}
template <int W>
__global__ void __launch_bounds__(128)
k_bits_count_csa(const u64 *__restrict__ X, u64 n, u64 ntiles, u32 *__restrict__ tc) {
    constexpr int WL = PullCfg<W>::WL, SPLIT = PullCfg<W>::SPLIT;
    const u32 lane = threadIdx.x & 31;
    const u64 wid = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const u64 tile = wid / SPLIT;
    const u32 h = (u32)(wid % SPLIT);
    if (tile >= ntiles) return;
    const u64 vbase = tile * TILE_V;
    // plane[p][w]: bit b = bit p of (number of this lane's 32 words of column w that have bit b set)
    u64 plane[6][WL];
    u64 pend[5][WL];            // carry waiting for its partner at level p + 1 (weight 2^(p+1))
#pragma unroll
    for (int p = 0; p < 6; p++)
#pragma unroll
        for (int w = 0; w < WL; w++) plane[p][w] = 0;
#pragma unroll
    for (int i = 0; i < 16; i++) {          // 16 pairs of vertices: v = lane + 32 * (2i), lane + 32 * (2i + 1)
        u64 xa[WL], xb[WL];
        const u64 va = vbase + lane + 64 * (u64)i, vb_ = va + 32;
        if (va < n) ld_part<WL>(xa, X + va * W + h * WL); else { for (int w = 0; w < WL; w++) xa[w] = 0; }
        if (vb_ < n) ld_part<WL>(xb, X + vb_ * W + h * WL); else { for (int w = 0; w < WL; w++) xb[w] = 0; }
#pragma unroll
        for (int w = 0; w < WL; w++) {
            u64 c;
            csa(c, plane[0][w], plane[0][w], xa[w], xb[w]);      // carry of weight 2
            // binary counter of pending carries: level L combines two carries of weight 2^L with the running plane
#pragma unroll
            for (int L = 1; L < 6; L++) {
                if ((i >> (L - 1)) & 1) {                        // second carry of this weight: combine, propagate
                    if (L < 5) { u64 c2; csa(c2, plane[L][w], plane[L][w], pend[L - 1][w], c); c = c2; }
                    else plane[5][w] ^= 0;                       // (unreachable: i < 16)
                } else { pend[L - 1][w] = c; break; }
            }
            if (i == 15) plane[5][w] = c;                        // the single carry of weight 32
        }
    }
    // planes -> counts: after transpose32 of one half-plane lane b holds bit b of all 32 lanes
#pragma unroll
    for (int w = 0; w < WL; w++) {
        u32 clo = 0, chi = 0;
#pragma unroll
        for (int p = 0; p < 6; p++) {
            clo += __popc(transpose32((u32)plane[p][w], lane)) << p;
            chi += __popc(transpose32((u32)(plane[p][w] >> 32), lane)) << p;
        }
        const u64 col = (u64)(h * WL + w) * 64;
        tc[(col + lane) * ntiles + tile] = clo;
        tc[(col + 32 + lane) * ntiles + tile] = chi;
    }
}

// Materialise fill.  A CTA owns a 1024-vertex tile (the count pass's tile) and reads each vertex record once: a pass loads
// G = min(W, 4) word columns of the tile's records -- 32 contiguous bytes per lane and vertex, one whole sector at W >= 4 --
// transposes them into a 64G x 32 mask tile in shared memory, and the warps then emit whole rows of that tile: lane l owns the
// 32 vertices of mask word l, a warp scan places the lanes (two rows per shuffle), the ids go to a warp-private u16 list aligned
// with the destination modulo 4 entries, and the list leaves as 16-byte stores with the tile's high id bits merged by PRMT.
// The mask tile is double-buffered and the next pass's records are loaded into registers before the rows are expanded, so one
// block barrier per pass separates the passes and the loads are in flight while the stores drain.  Loading one 8-byte word
// column per pass instead fetches every 32-byte sector up to four times and leaves loads and stores in separate phases: that is
// what bounded the fill (the id expansion itself is under 3 % of its time).  64 registers and ~98 KB of shared memory: 2 CTAs per SM.
template <int W> struct FillCfg {
    static constexpr u32 G = W < 4 ? W : 4;       // word columns per pass
    static constexpr u32 NP = W / G;              // passes per tile
    static constexpr u32 ROWS = 64 * G;           // mask rows per pass
};
static const u32 FILL_STRIDE = 33;                          // padded row stride of the mask tile (bank-conflict free)
static const u32 FILL_LIST = TILE_V + 8;                    // entries per warp list (+3 alignment slack, rounded)
template <int W> constexpr size_t fill_smem() {
    return 2 * FillCfg<W>::ROWS * FILL_STRIDE * sizeof(u32) + (TILE_THREADS / 32) * FILL_LIST * sizeof(unsigned short);
}
template <int G> __device__ __forceinline__ void ld_words(u64 (&x)[G], const u64 *p) {
    if constexpr (G == 1) { x[0] = __ldg(p); }
    else {
#pragma unroll
        for (int k = 0; k < G; k += 2) { ulonglong2 q = __ldg(reinterpret_cast<const ulonglong2 *>(p) + k / 2); x[k] = q.x; x[k + 1] = q.y; }
    }
}
template <int W>
__global__ void __launch_bounds__(TILE_THREADS, 2)
k_bits_fill(const u64 *__restrict__ X, u64 n, u64 ntiles, const u64 *__restrict__ off, u32 *__restrict__ Cj) {
    using Cfg = FillCfg<W>;
    constexpr u32 G = Cfg::G, NP = Cfg::NP, ROWS = Cfg::ROWS, NW = TILE_THREADS / 32, RPW = ROWS / NW;
    static_assert(RPW % 4 == 0, "rows are scanned in groups of four");
    extern __shared__ __align__(16) unsigned char fill_smem_raw[];
    u32 *T = reinterpret_cast<u32 *>(fill_smem_raw);                                // [2][ROWS][FILL_STRIDE]
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    unsigned short *L = reinterpret_cast<unsigned short *>(fill_smem_raw + 2 * ROWS * FILL_STRIDE * sizeof(u32)) + warp * FILL_LIST;
    const u64 strm = policy_stream();
    const u64 tile = blockIdx.x;
    const u64 vbase = tile * TILE_V;
    const u32 lo16base = (u32)(vbase & 0xFFFFu), vbhi = (u32)(vbase >> 16);     // a 1024-aligned tile never crosses 2^16
    u64 x[2][G];
#pragma unroll
    for (u32 g = 0; g < 2; g++) {
        const u64 v = vbase + (u64)warp * 64 + g * 32 + lane;
        if (v < n) ld_words<G>(x[g], X + v * W);
        else {
#pragma unroll
            for (u32 k = 0; k < G; k++) x[g][k] = 0;
        }
    }
    for (u32 p = 0; p < NP; p++) {
        u32 *Tp = T + (p & 1) * ROWS * FILL_STRIDE;
#pragma unroll
        for (u32 g = 0; g < 2; g++) {
#pragma unroll
            for (u32 k = 0; k < G; k++) {
                u32 tl = 0, th = 0;
                if (__ballot_sync(0xffffffffu, x[g][k] != 0ULL)) {
                    tl = transpose32((u32)x[g][k], lane);
                    th = transpose32((u32)(x[g][k] >> 32), lane);
                }
                Tp[(k * 64 + lane) * FILL_STRIDE + 2 * warp + g] = tl;
                Tp[(k * 64 + 32 + lane) * FILL_STRIDE + 2 * warp + g] = th;
            }
        }
        if (p + 1 < NP) {                               // next pass's words in flight during this pass's expansion
#pragma unroll
            for (u32 g = 0; g < 2; g++) {
                const u64 v = vbase + (u64)warp * 64 + g * 32 + lane;
                if (v < n) ld_words<G>(x[g], X + v * W + (p + 1) * G);
            }
        }
        __syncthreads();
        // rows of this pass: r = warp + NW * i; row r is frontier row 64 * (p * G) + r
        const u64 obase = (u64)p * ROWS;
#pragma unroll 1
        for (u32 i0 = 0; i0 < RPW; i0 += 4) {
            u64 g0[4];
#pragma unroll
            for (u32 i = 0; i < 4; i++) g0[i] = off[(obase + warp + NW * (i0 + i)) * ntiles + tile];
            u32 m[4], c[4];
#pragma unroll
            for (u32 i = 0; i < 4; i++) { m[i] = Tp[(warp + NW * (i0 + i)) * FILL_STRIDE + lane]; c[i] = __popc(m[i]); }
            u32 pk[2] = {c[0] | (c[1] << 16), c[2] | (c[3] << 16)};          // prefixes stay below 2^16 (tile = 1024)
#pragma unroll
            for (u32 d = 1; d < 32; d <<= 1) {
#pragma unroll
                for (u32 h = 0; h < 2; h++) { const u32 t = __shfl_up_sync(0xffffffffu, pk[h], d); if (lane >= d) pk[h] += t; }
            }
#pragma unroll
            for (u32 i = 0; i < 4; i++) {
                const u32 field = (i & 1) ? (pk[i / 2] >> 16) : (pk[i / 2] & 0xFFFFu);
                const u32 cnt = __shfl_sync(0xffffffffu, field, 31);
                if (cnt == 0) continue;
                const u32 a = (u32)(g0[i] & 3);
                u32 o = a + field - c[i];
                const u32 idb = lo16base + lane * 32;
                u32 mm = m[i];
                while (mm) { const u32 bit = __ffs(mm) - 1; L[o++] = (unsigned short)(idb + bit); mm &= mm - 1; }
                __syncwarp();
                u32 *dst = Cj + (g0[i] - a);                // 16-byte aligned; dst[k] <-> L[k] for k in [a, a + cnt)
                const u32 total = a + cnt;
                const u32 head_end = a ? (total < 4 ? total : 4) : 0;
                if (lane >= a && lane < head_end) st_u32_stream(dst + lane, (vbhi << 16) | L[lane], strm);
                const u32 nfull = total >> 2;
                const uint2 *L2 = reinterpret_cast<const uint2 *>(L);
                uint4 *dv = reinterpret_cast<uint4 *>(dst);
                for (u32 k = (a ? 1 : 0) + lane; k < nfull; k += 32) {
                    const uint2 q2 = L2[k];
                    uint4 q;
                    q.x = __byte_perm(q2.x, vbhi, 0x5410); q.y = __byte_perm(q2.x, vbhi, 0x5432);
                    q.z = __byte_perm(q2.y, vbhi, 0x5410); q.w = __byte_perm(q2.y, vbhi, 0x5432);
                    __stcs(dv + k, q);
                }
                const u32 tail = nfull * 4 > head_end ? nfull * 4 : head_end;
                if (tail + lane < total) st_u32_stream(dst + tail + lane, (vbhi << 16) | L[tail + lane], strm);
                __syncwarp();
            }
        }
    }
}

__global__ void k_bits_rowptr(const u64 *__restrict__ off, u64 nrows, u64 ntiles, u64 *__restrict__ Cp) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r <= nrows) Cp[r] = off[r * ntiles];
}

template <int W> static void launch_fill(const DevBits &X, u64 ntiles, const u64 *off, u32 *Cj) {
    static bool attr_set = false;
    if (!attr_set) {
        CUDA_TRY(cudaFuncSetAttribute(k_bits_fill<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fill_smem<W>()));
        attr_set = true;
    }
    LAUNCH(k_bits_fill<W>, (u32)ntiles, TILE_THREADS, fill_smem<W>(), X.w.ptr, X.ncols, ntiles, off, Cj);
}

void bits_to_csr(const DevBits &X, DevCSR &C) {
    require_natural(X, "bits_to_csr");
    u64 n = X.ncols;
    u32 W = X.W;
    C.clear();
    C.nrows = X.nrows; C.ncols = n;
    C.p.alloc(X.nrows + 1);
    if (n == 0) { C.p.zero(); C.nnz = 0; return; }
    u64 ntiles = (n + TILE_V - 1) / TILE_V;
    u64 ncnt = (u64)64 * W * ntiles;
    DevBuf<u32> tc(ncnt + 1);
    DevBuf<u64> off(ncnt + 1);
    {
        TimedScope ts(TK_BITS_COUNT, 8ULL * W * n);
        const u64 nwarps = ntiles * pull_split((int)W);
        const u32 g = (u32)((nwarps + 3) / 4);
        switch (W) {
        case 1: LAUNCH((k_bits_count_csa<1>), g, 128, 0, X.w.ptr, n, ntiles, tc.ptr); break;
        case 2: LAUNCH((k_bits_count_csa<2>), g, 128, 0, X.w.ptr, n, ntiles, tc.ptr); break;
        case 4: LAUNCH((k_bits_count_csa<4>), g, 128, 0, X.w.ptr, n, ntiles, tc.ptr); break;
        case 8: LAUNCH((k_bits_count_csa<8>), g, 128, 0, X.w.ptr, n, ntiles, tc.ptr); break;
        default: LAUNCH((k_bits_count_csa<16>), g, 128, 0, X.w.ptr, n, ntiles, tc.ptr); break;
        }
    }
    CUDA_TRY(cudaMemsetAsync(tc.ptr + ncnt, 0, sizeof(u32), stream()));
    exclusive_scan_u32_to_u64(tc.ptr, off.ptr, ncnt + 1);
    LAUNCH(k_bits_rowptr, grid_for(X.nrows + 1, 256), 256, 0, off.ptr, X.nrows, ntiles, C.p.ptr);
    u64 nnz = read_scalar(off.ptr + X.nrows * ntiles);
    C.nnz = nnz;
    C.j.alloc(nnz);
    if (nnz) {
        TimedScope ts(TK_BITS_FILL, 8ULL * W * n + 4 * nnz);
        switch (W) {
        case 1: launch_fill<1>(X, ntiles, off.ptr, C.j.ptr); break;
        case 2: launch_fill<2>(X, ntiles, off.ptr, C.j.ptr); break;
        case 4: launch_fill<4>(X, ntiles, off.ptr, C.j.ptr); break;
        case 8: launch_fill<8>(X, ntiles, off.ptr, C.j.ptr); break;
        default: launch_fill<16>(X, ntiles, off.ptr, C.j.ptr); break;
        }
    }
}

// ---------------------------------------------------------------------------- diagonal operand = column filter
// Label matrices are n x n diagonal (graph.rs:1191): F * L keeps column j of F iff L(j,j) is present -- an elementwise pass
// over the bit-matrix instead of a hop (SURVEY 8f-2, label-filter fusion).
__global__ void __launch_bounds__(256) k_is_diagonal(const u64 *__restrict__ p, const u32 *__restrict__ j, u64 n, u32 *__restrict__ bad) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    bool b = false;
    for (; r < n; r += stride) {
        u64 s = p[r], e = p[r + 1];
        if (e - s > 1 || (e - s == 1 && j[s] != (u32)r)) b = true;
    }
    if (__any_sync(0xffffffffu, b) && (threadIdx.x & 31) == 0) atomicOr(bad, 1u);
}
bool csr_is_diagonal(const DevCSR &A) {
    if (A.nrows != A.ncols || A.nnz > A.nrows) return false;
    if (A.nrows == 0) return true;
    DevBuf<u32> bad(1);
    bad.zero();
    LAUNCH(k_is_diagonal, grid_for(A.nrows, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, A.j.ptr, A.nrows, bad.ptr);
    return read_scalar(bad.ptr) == 0;
}
__global__ void __launch_bounds__(256)
k_bits_diag(const u64 *__restrict__ X, const u64 *__restrict__ Ap, u64 n, u32 W, u64 *__restrict__ Y, u64 *__restrict__ flops) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x, total = n * W;
    u64 c = 0;
    for (; t < total; t += stride) {
        const u64 v = t / W;
        const u64 x = (Ap[v + 1] > Ap[v]) ? X[t] : 0ULL;
        Y[t] = x;
        c += __popcll(x);
    }
    u64 tot = Red(ts).Sum(c);
    if (threadIdx.x == 0 && tot) atomicAdd((unsigned long long *)flops, tot);
}
void bits_diag(const DevBits &X, const DevCSR &A, DevBits &Y, u64 *flops_out) {
    require_natural(X, "bits_diag");
    if (X.ncols != A.nrows) throw GrbError(-6, "mxm: inner dimensions differ");
    Y.clear();
    Y.nrows = X.nrows; Y.ncols = A.ncols; Y.W = X.W;
    Y.w.alloc(A.ncols * X.W);
    DevBuf<u64> fl(1);
    fl.zero();
    if (A.nrows) LAUNCH(k_bits_diag, grid_for(A.nrows * X.W, 256, (u64)ctx().num_sms * 16), 256, 0, X.w.ptr, A.p.ptr, A.nrows, X.W, Y.w.ptr, fl.ptr);
    if (flops_out) *flops_out = read_scalar(fl.ptr);
}

// ---------------------------------------------------------------------------- row-major bitmap (GxB_BITMAP-like export)
// out[row * wpr + (v >> 6)] bit (v & 63) <=> X(row, v).  Same 64 x 1024 transposed tile as the materialise kernels, written
// out as 128-byte row segments; rows >= nrows (padding of the last word column) are dropped.
__global__ void __launch_bounds__(TILE_THREADS)
k_bits_rowmajor(const u64 *__restrict__ X, u64 n, u32 W, u64 nrows, u64 wpr, u64 *__restrict__ out) {
    __shared__ u32 T[2][64 * FILL_STRIDE];
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u64 tile = blockIdx.x;
    const u64 vbase = tile * TILE_V;
    const u64 strm = policy_stream();
    for (u32 w = 0; w < W; w++) {
        if ((u64)w * 64 >= nrows) break;
        u32 *Tw = T[w & 1];
#pragma unroll
        for (u32 g = 0; g < 2; g++) {
            u64 v = vbase + (u64)warp * 64 + g * 32 + lane;
            u64 word = (v < n) ? X[v * W + w] : 0ULL;
            u32 tl = 0, th = 0;
            if (__ballot_sync(0xffffffffu, word != 0ULL)) {
                tl = transpose32((u32)word, lane);
                th = transpose32((u32)(word >> 32), lane);
            }
            Tw[lane * FILL_STRIDE + 2 * warp + g] = tl;
            Tw[(lane + 32) * FILL_STRIDE + 2 * warp + g] = th;
        }
        __syncthreads();
#pragma unroll
        for (u32 h = 0; h < 2; h++) {
            u32 r = (tid >> 4) + 32 * h, c = tid & 15;
            u64 row = (u64)w * 64 + r, col = tile * (TILE_V / 64) + c;
            if (row < nrows && col < wpr) {
                u64 val = (u64)Tw[r * FILL_STRIDE + 2 * c] | ((u64)Tw[r * FILL_STRIDE + 2 * c + 1] << 32);
                st_u64_stream(out + row * wpr + col, val, strm);
            }
        }
    }
}

void bits_to_rowmajor(const DevBits &X, u64 *out, u64 wpr) {
    require_natural(X, "bits_to_rowmajor");
    u64 n = X.ncols;
    if (!n || !X.nrows) return;
    u64 ntiles = (n + TILE_V - 1) / TILE_V;
    LAUNCH(k_bits_rowmajor, (u32)ntiles, TILE_THREADS, 0, X.w.ptr, n, X.W, X.nrows, wpr, out);
}

// CSR -> row-major bitmap for matrices that are not in frontier form (out must be zeroed); one warp per row
__global__ void k_csr_to_bitmap(const u64 *__restrict__ p, const u32 *__restrict__ j, u64 nrows, u64 wpr, u64 *__restrict__ out) {
    u64 row = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u32 lane = threadIdx.x & 31;
    if (row >= nrows) return;
    for (u64 q = p[row] + lane; q < p[row + 1]; q += 32) {
        u32 c = j[q];
        atomicOr((unsigned long long *)(out + row * wpr + (c >> 6)), 1ULL << (c & 63));
    }
}
void csr_to_rowmajor(const DevCSR &A, u64 *out, u64 wpr) {
    if (!A.nrows || !A.nnz) return;
    LAUNCH(k_csr_to_bitmap, grid_for(A.nrows * 32, 256), 256, 0, A.p.ptr, A.j.ptr, A.nrows, wpr, out);
}

// ---------------------------------------------------------------------------- reductions
__global__ void __launch_bounds__(256) k_popc_sum(const u64 *__restrict__ w, u64 n, u64 *__restrict__ out) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 s = 0;
    for (; t < n; t += stride) s += __popcll(w[t]);
    u64 tot = Red(ts).Sum(s);
    if (threadIdx.x == 0 && tot) atomicAdd((unsigned long long *)out, tot);
}

u64 bits_nvals(const DevBits &X) {
    DevBuf<u64> out(1);
    out.zero();
    u64 n = X.ncols * X.W;
    if (n) LAUNCH(k_popc_sum, grid_for(n, 256, (u64)ctx().num_sms * 8), 256, 0, X.w.ptr, n, out.ptr);
    return read_scalar(out.ptr);
}

// flops (mxm sense) = sum_k popc(X[k]) * deg_A(k); edges = sum_{k active} deg_A(k); flag[k] = active
__global__ void __launch_bounds__(256)
k_bits_flops(const u64 *__restrict__ X, u32 W, u64 n, const u64 *__restrict__ Ap, u32 *__restrict__ flag,
             u64 *__restrict__ out /* [0]=flops [1]=edges */) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts, ts2;
    u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 fl = 0, ed = 0;
    for (; k < n; k += stride) {
        u32 pc = 0;
        for (u32 w = 0; w < W; w++) pc += __popcll(X[k * W + w]);
        u64 d = Ap[k + 1] - Ap[k];
        flag[k] = (pc != 0 && d != 0) ? 1u : 0u;
        if (pc) { fl += (u64)pc * d; ed += d; }
    }
    u64 tf = Red(ts).Sum(fl);
    u64 te = Red(ts2).Sum(ed);
    if (threadIdx.x == 0) {
        if (tf) atomicAdd((unsigned long long *)&out[0], tf);
        if (te) atomicAdd((unsigned long long *)&out[1], te);
    }
}

// ---------------------------------------------------------------------------- push
__global__ void k_compact_active(const u32 *__restrict__ flag, const u64 *__restrict__ pos, u64 n,
                                 const u64 *__restrict__ Ap, u32 *__restrict__ act, u64 *__restrict__ deg,
                                 u64 *__restrict__ astart) {
    u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; k < n; k += stride) {
        if (flag[k]) {
            u64 d = pos[k];
            act[d] = (u32)k;
            u64 s = Ap[k];
            deg[d] = Ap[k + 1] - s;
            astart[d] = s;
        }
    }
}

__device__ __forceinline__ u64 find_le64(const u64 *__restrict__ a, u64 lo, u64 hi, u64 target) {
    while (lo < hi) {
        u64 mid = (lo + hi + 1) >> 1;
        if (a[mid] <= target) lo = mid; else hi = mid - 1;
    }
    return lo;
}

template <int W>
__global__ void __launch_bounds__(256)
k_bits_push(const u32 *__restrict__ act, const u64 *__restrict__ cum, const u64 *__restrict__ astart, u64 nact,
            u64 total, const u32 *__restrict__ Aj, const u64 *__restrict__ X, u64 *__restrict__ Y) {
    __shared__ u64 s_e0, s_e1;
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    u64 lo = (u64)blockIdx.x * PUSH_CHUNK, hi = lo + PUSH_CHUNK;
    if (hi > total) hi = total;
    if (tid == 0) {
        s_e0 = find_le64(cum, 0, nact - 1, lo);
        s_e1 = find_le64(cum, 0, nact - 1, hi - 1);
    }
    __syncthreads();
    u64 e0 = s_e0, e1 = s_e1;
    for (u64 t0 = lo + (u64)warp * 32; t0 < hi; t0 += 8 * 32) {
        u64 e = find_le64(cum, e0, e1, t0);
        u64 t = t0 + lane;
        if (t < hi) {
            while (e < e1 && cum[e + 1] <= t) e++;
            u32 k = act[e];
            u32 col = Aj[astart[e] + (t - cum[e])];
#pragma unroll
            for (int w = 0; w < W; w++) {
                u64 xw = X[(u64)k * W + w];
                if (xw) atomicOr((unsigned long long *)&Y[(u64)col * W + w], xw);
            }
        }
    }
}

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
// ANDNOT (the dirty hop's deleted-edge term, bits_apply_deltas) clears bit i instead of setting it.  SLICED (csr_push_sliced): the
// entries are sub-entries, Ap[e] is where sub-entry e starts in Aj, Fj is not read, and a CTA takes CHUNK flops.
template <int W, bool ANDNOT, bool SLICED = false, u64 CHUNK = PUSH_CHUNK>
__global__ void __launch_bounds__(256)
k_csr_push(const u32 *__restrict__ erow, const u32 *__restrict__ Fj, const u64 *__restrict__ cum, u64 nent, u64 total,
           const u64 *__restrict__ Ap, const u32 *__restrict__ Aj, u64 *__restrict__ Y, const u32 *__restrict__ perm) {
    __shared__ u64 s_e0, s_e1;
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    u64 lo = (u64)blockIdx.x * CHUNK, hi = lo + CHUNK;
    if (hi > total) hi = total;
    if (tid == 0) {
        s_e0 = find_le64(cum, 0, nent - 1, lo);
        s_e1 = find_le64(cum, 0, nent - 1, hi - 1);
    }
    __syncthreads();
    u64 e0 = s_e0, e1 = s_e1;
    for (u64 t0 = lo + (u64)warp * 32; t0 < hi; t0 += 8 * 32) {
        u64 e = find_le64(cum, e0, e1, t0);
        u64 t = t0 + lane;
        if (t < hi) {
            while (e < e1 && cum[e + 1] <= t) e++;
            const u32 i = erow[e];
            u32 col = Aj[(SLICED ? Ap[e] : Ap[Fj[e]]) + (t - cum[e])];
            // hot-set order through the table (the deltas, which have no relabelled copy); a prepared operand passes its
            // relabelled col_idx (PullTables::ap) as Aj instead, with perm null
            if (perm) col = __ldg(perm + col);
            unsigned long long *dst = (unsigned long long *)&Y[(u64)col * W + (i >> 6)];
            if (ANDNOT) atomicAnd(dst, ~(1ULL << (i & 63)));
            else atomicOr(dst, 1ULL << (i & 63));
        }
    }
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
    if (F.nnz) {
        DevBuf<u32> seen((F.ncols + 31) / 32);
        seen.zero();
        CUDA_TRY(cudaMemsetAsync(cum.ptr + F.nnz, 0, 2 * sizeof(u64), stream()));
        LAUNCH(k_csr_entry_info, grid_for(F.nrows * 32, 256), 256, 0, F.p.ptr, F.j.ptr, F.nrows, A.p.ptr, erow.ptr, cum.ptr, seen.ptr,
               cum.ptr + F.nnz + 1);
        exclusive_scan_u64(cum.ptr, cum.ptr, F.nnz + 1);
        u64 h[2];
        d2h(h, cum.ptr + F.nnz, 2);
        sync_stream();
        flops = h[0]; edges = h[1];
    }
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
    if (P) {
        switch (W) {
        case 1: csr_push_sliced<1>(F, A, Aj, Y, flops, erow.ptr, P, S); break;
        case 2: csr_push_sliced<2>(F, A, Aj, Y, flops, erow.ptr, P, S); break;
        case 4: csr_push_sliced<4>(F, A, Aj, Y, flops, erow.ptr, P, S); break;
        case 8: csr_push_sliced<8>(F, A, Aj, Y, flops, erow.ptr, P, S); break;
        default: csr_push_sliced<16>(F, A, Aj, Y, flops, erow.ptr, P, S); break;
        }
        return true;
    }
    switch (W) {
    case 1: csr_push_impl<1>(F, A, Aj, Y, flops, erow.ptr, cum.ptr, perm, acc); break;
    case 2: csr_push_impl<2>(F, A, Aj, Y, flops, erow.ptr, cum.ptr, perm, acc); break;
    case 4: csr_push_impl<4>(F, A, Aj, Y, flops, erow.ptr, cum.ptr, perm, acc); break;
    case 8: csr_push_impl<8>(F, A, Aj, Y, flops, erow.ptr, cum.ptr, perm, acc); break;
    default: csr_push_impl<16>(F, A, Aj, Y, flops, erow.ptr, cum.ptr, perm, acc); break;
    }
    return true;
}

// permuted form -> natural order: Xn[pvert[s]] = X[s], one thread per word
__global__ void k_unpermute(const u64 *__restrict__ X, const u32 *__restrict__ pvert, u64 n, u32 W, u64 *__restrict__ out) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x, total = n * W;
    for (; t < total; t += stride) { const u64 s = t / W, w = t - s * W; out[(u64)pvert[s] * W + w] = X[t]; }
}
void bits_naturalise(DevBits &X) {
    if (!X.permuted()) return;
    const u64 n = X.ncols;
    DevBuf<u64> out(n * X.W);
    if (n) LAUNCH(k_unpermute, grid_for(n * X.W, 256, (u64)ctx().num_sms * 32), 256, 0, X.w.ptr, X.pvert->ptr, n, X.W, out.ptr);
    X.w = std::move(out);
    X.pvert.reset();
    X.pperm.reset();
    X.perm_tag = 0;
}
static void require_natural(const DevBits &X, const char *what) {
    if (X.permuted()) throw GrbError(-101, std::string(what) + ": frontier is in permuted form (internal error: bits_naturalise was not called)");
}

// ---------------------------------------------------------------------------- pull
// Y[j] = OR of X[k] over k in A'(j,:).  What bounds a pull is the L1TEX tag stage: one 128-byte line per clock per SM, and a
// warp-wide gather with every lane on a different vertex costs 32 of those "wavefronts" per instruction.  A vertex record of
// W = 8 words is 64 bytes -- one line -- but a lane can fetch at most 16 bytes per instruction on sm_90 (LDG.128), so
// one-lane-per-vertex spends FOUR wavefronts per vertex.  In k_pull_seg SPLIT = W / 2 adjacent lanes share a vertex: lane h loads
// words [2h, 2h+2) of the record with one LDG.128, the requests fall into the same line and coalesce into one wavefront, and the
// lanes never exchange data (each lane ORs, keeps and finally stores its own 16-byte part of the output row).
// W = 4 -> half the wavefronts per gathered vertex; W = 8 -> a quarter; W = 16 -> an eighth; W <= 2 keeps one lane per record.
// The rows of A' are binned once per matrix (build_pull_tables):
//   small (<= SMALL_ROW entries) : k_pull_small, one lane per row in natural order; it also zero-fills the long rows
//   mid   (<= LONG_ROW)          : k_pull_seg, 8 lanes per row, from a list sorted by length, descending
//   long                         : the same list, as LONG_ROW-entry segments whose partial results are merged with RED.OR
struct OrOp64 { __device__ u64 operator()(u64 a, u64 b) const { return a | b; } };

// G[w] = OR over all vertices of word w: the terminal value of the OR monoid for this frontier.  A pull row whose
// accumulator has reached G cannot change any more, so the rest of its neighbours need not be gathered (exact).
template <int W>
__global__ void __launch_bounds__(256) k_or_all(const u64 *__restrict__ X, u64 nv, u64 *__restrict__ G) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 acc[W];
#pragma unroll
    for (int w = 0; w < W; w++) acc[w] = 0;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < nv; t += stride) {
#pragma unroll
        for (int w = 0; w < W; w++) acc[w] |= X[t * W + w];
    }
#pragma unroll
    for (int w = 0; w < W; w++) {
        u64 r = Red(ts).Reduce(acc[w], OrOp64());
        __syncthreads();
        if (threadIdx.x == 0 && r) atomicOr((unsigned long long *)&G[w], r);
    }
}

// The L2 policies of one pull launch with hints on.  The gather source X (the packed frontier, hot-set order: out-degree
// descending) is evict_last over its first `hot` bytes and evict_first over the rest of its `tot` bytes, or evict_normal
// everywhere when hot = 0.  streams != 0: A' col_idx and rowptr, the segment list and the stores of Y are evict_first, so the
// 2 GB that pass through once do not push the hot records out.
struct PullHints {
    u32 hot = 0, tot = 0, streams = 0;
#ifdef __CUDACC__
    __device__ __forceinline__ u64 gather_policy(const void *X) const { return hot ? policy_range(X, hot, tot) : policy_normal(); }
    __device__ __forceinline__ u64 stream_policy() const { return streams ? policy_stream() : policy_normal(); }
#endif
};

// HINTS: every load of the pull kernels carries an L2 policy (PullHints).  A' col_idx and rowptr lines are shared by the loads of
// neighbouring lanes and unroll steps, so they keep their L1 allocation; only their L2 priority changes
template <bool HINTS> __device__ __forceinline__ u32 ld_col(const u32 *p, u64 strm) { return HINTS ? ld_nc_u32(p, strm) : __ldg(p); }
template <bool HINTS> __device__ __forceinline__ u64 ld_ptr(const u64 *p, u64 strm) { return HINTS ? ld_nc_u64(p, strm) : __ldg(p); }
template <bool HINTS> __device__ __forceinline__ u64 ld_x(const u64 *p, u64 keep) { return HINTS ? ld_nc_u64(p, keep) : __ldg(p); }
// acc |= the W frontier words of one vertex: ONE 16-byte load per word pair (a W=4 vertex is a single 32 B sector), so the
// number of L1TEX wavefronts per gathered vertex does not grow with W
template <int W, bool HINTS> __device__ __forceinline__ void or_words(u64 (&acc)[W], const u64 *__restrict__ p, u64 keep) {
    if (W == 1) { acc[0] |= ld_x<HINTS>(p, keep); return; }
    const ulonglong2 *q = reinterpret_cast<const ulonglong2 *>(p);
#pragma unroll
    for (int w2 = 0; w2 < W / 2; w2++) {
        ulonglong2 v = HINTS ? ld_nc_v2(q + w2, keep) : __ldg(q + w2);
        acc[2 * w2] |= v.x;
        acc[2 * w2 + 1] |= v.y;
    }
}

static const u32 SMALL_ROW = 8;

// HINTS: the store carries policy pol (Y is written once and read by the next pass, not by this kernel)
template <int W, bool HINTS = false> __device__ __forceinline__ void store_row(u64 *dst, const u64 (&acc)[W], u64 pol = 0) {
    if constexpr (W == 1) {
        if (HINTS) st_u64_stream(dst, acc[0], pol);
        else dst[0] = acc[0];
    } else {
#pragma unroll
        for (int w2 = 0; w2 < W / 2; w2++) {
            ulonglong2 *q = reinterpret_cast<ulonglong2 *>(dst) + w2;
            if (HINTS) st_v2_hint(q, make_ulonglong2(acc[2 * w2], acc[2 * w2 + 1]), pol);
            else *q = make_ulonglong2(acc[2 * w2], acc[2 * w2 + 1]);
        }
    }
}
template <int WL, bool HINTS = false> __device__ __forceinline__ void store_part(u64 *dst, const u64 (&acc)[WL], u64 pol = 0) {
    store_row<WL, HINTS>(dst, acc, pol);
}
// accumulate mode (union hops): dst |= acc, skipped when acc is empty.  Each record is owned by one lane (k_pull_small) or one
// 8-lane group (a mid row of k_pull_seg), so a plain read-modify-write is race-free
template <int WL> __device__ __forceinline__ void or_part(u64 *dst, u64 (&acc)[WL]) {
    u64 any = 0;
#pragma unroll
    for (int w = 0; w < WL; w++) any |= acc[w];
    if (!any) return;
    if constexpr (WL == 1) { dst[0] |= acc[0]; }
    else {
#pragma unroll
        for (int w2 = 0; w2 < WL / 2; w2++) {
            ulonglong2 v = reinterpret_cast<const ulonglong2 *>(dst)[w2];
            reinterpret_cast<ulonglong2 *>(dst)[w2] = make_ulonglong2(v.x | acc[2 * w2], v.y | acc[2 * w2 + 1]);
        }
    }
}

static const u32 SEG_ATOMIC = 0x80000000u;

// segments per row: 0 (small), 1 (mid), ceil(len / LONG_ROW) (long); maxlen = the longest row when it is longer than LONG_ROW
__global__ void k_seg_count(const u64 *__restrict__ p, u64 n, u32 *__restrict__ cnt, u64 *__restrict__ maxlen) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 mx = 0;
    for (; r <= n; r += stride) {
        if (r == n) { cnt[r] = 0; break; }
        u64 d = p[r + 1] - p[r];
        cnt[r] = d <= SMALL_ROW ? 0u : (u32)((d + LONG_ROW - 1) / LONG_ROW);
        if (d > mx) mx = d;
    }
    if (mx > LONG_ROW) atomicMax((unsigned long long *)maxlen, mx);
}
// key = LONG_ROW - seglen (ascending sort = longest first), value = position of the segment: row << 20 | index inside the row
__global__ void k_seg_emit(const u64 *__restrict__ p, u64 n, const u64 *__restrict__ pos, u64 *__restrict__ keys, u64 *__restrict__ vals) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; r < n; r += stride) {
        const u64 d = p[r + 1] - p[r];
        if (d <= SMALL_ROW) continue;
        u64 o = pos[r];
        for (u64 s = 0, i = 0; s < d; s += LONG_ROW, i++) {
            const u64 len = d - s < LONG_ROW ? d - s : LONG_ROW;
            keys[o] = LONG_ROW - len;
            vals[o] = (r << 20) | i;
            o++;
        }
    }
}
__global__ void k_seg_unpack(const u64 *__restrict__ vals, u64 ns, const u64 *__restrict__ p, u32 *__restrict__ s_row,
                             u32 *__restrict__ s_len, u64 *__restrict__ s_start) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ns) return;
    const u64 v = vals[i];
    const u32 r = (u32)(v >> 20);
    const u64 k = v & 0xFFFFFu;
    const u64 d = p[r + 1] - p[r];
    const u64 s = k * LONG_ROW;
    const u64 len = d - s < LONG_ROW ? d - s : LONG_ROW;
    s_row[i] = r;
    s_start[i] = p[r] + s;
    s_len[i] = (u32)len | (d > LONG_ROW ? SEG_ATOMIC : 0u);
}
static void build_seg_list(const DevCSR &AT, PullTables &pt) {
    const u64 n = AT.nrows;
    pt.ns = 0;
    pt.s_row.release(); pt.s_len.release(); pt.s_start.release();
    if (!n) return;
    DevBuf<u32> cnt(n + 1);
    DevBuf<u64> pos(n + 1), mx(1);
    mx.zero();
    LAUNCH(k_seg_count, grid_for(n + 1, 256, 1 << 16), 256, 0, AT.p.ptr, n, cnt.ptr, mx.ptr);
    // k_seg_emit addresses a segment as row << 20 | index inside the row
    if (read_scalar(mx.ptr) >= ((u64)LONG_ROW << 20)) throw GrbError(-8, "pull: a row of A' exceeds 2^32 entries");
    exclusive_scan_u32_to_u64(cnt.ptr, pos.ptr, n + 1);
    const u64 ns = read_scalar(pos.ptr + n);
    pt.ns = ns;
    if (!ns) return;
    DevBuf<u64> keys(ns), vals(ns);
    LAUNCH(k_seg_emit, grid_for(n, 256, 1 << 16), 256, 0, AT.p.ptr, n, pos.ptr, keys.ptr, vals.ptr);
    sort_pairs_u64(keys.ptr, vals.ptr, ns, 13);          // stable: rows ascending inside one length
    pt.s_row.alloc(ns); pt.s_len.alloc(ns); pt.s_start.alloc(ns);
    LAUNCH(k_seg_unpack, grid_for(ns, 256), 256, 0, vals.ptr, ns, AT.p.ptr, pt.s_row.ptr, pt.s_len.ptr, pt.s_start.ptr);
}

// one lane per row, natural order: rows of <= SMALL_ROW entries are finished here, rows longer than LONG_ROW are zero-filled
// (their segments arrive through RED.OR), everything in between is left to k_pull_seg.  This kernel is latency-bound, not
// L1TEX-bound: splitting the record across lanes as k_pull_seg does would divide the bytes each warp keeps in flight, so one lane
// owns the whole record here.  ACC (union hops): Y already holds earlier operands' products; small rows are ORed into it and long
// rows are left as they are.
template <int W, bool HINTS, bool ACC>
__global__ void __launch_bounds__(256)
k_pull_small(const u64 *__restrict__ ATp, const u32 *__restrict__ ATj, u64 n, const u64 *__restrict__ X,
             u64 *__restrict__ Y, PullHints ph) {
    const u64 keep = HINTS ? ph.gather_policy(X) : 0, strm = HINTS ? ph.stream_policy() : 0;
    u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    // three-stage pipeline per lane: row pointers two rows ahead, first col_idx batch one row ahead, gathers now
    u64 s = 0, e = 0, s1 = 0, e1 = 0;
    if (j < n) { s = ld_ptr<HINTS>(ATp + j, strm); e = ld_ptr<HINTS>(ATp + j + 1, strm); }
    if (j + stride < n) { s1 = ld_ptr<HINTS>(ATp + j + stride, strm); e1 = ld_ptr<HINTS>(ATp + j + stride + 1, strm); }
    u32 k[4];
#pragma unroll
    for (int u = 0; u < 4; u++) k[u] = (e - s <= SMALL_ROW && s + u < e) ? ld_col<HINTS>(ATj + s + u, strm) : 0xFFFFFFFFu;
    for (; j < n; j += stride) {
        u64 s2 = 0, e2 = 0;
        if (j + 2 * stride < n) { s2 = ld_ptr<HINTS>(ATp + j + 2 * stride, strm); e2 = ld_ptr<HINTS>(ATp + j + 2 * stride + 1, strm); }
        u32 kn[4];
#pragma unroll
        for (int u = 0; u < 4; u++) kn[u] = (e1 - s1 <= SMALL_ROW && s1 + u < e1) ? ld_col<HINTS>(ATj + s1 + u, strm) : 0xFFFFFFFFu;
        u64 acc[W];
#pragma unroll
        for (int w = 0; w < W; w++) acc[w] = 0;
        if (e - s <= SMALL_ROW) {
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (k[u] != 0xFFFFFFFFu) or_words<W, HINTS>(acc, X + (u64)k[u] * W, keep);
            if (e - s > 4) {
#pragma unroll
                for (int u = 0; u < 4; u++) k[u] = (s + 4 + u < e) ? ld_col<HINTS>(ATj + s + 4 + u, strm) : 0xFFFFFFFFu;
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (k[u] != 0xFFFFFFFFu) or_words<W, HINTS>(acc, X + (u64)k[u] * W, keep);
            }
        }
        if (ACC) { if (e - s <= SMALL_ROW) or_part<W>(Y + j * W, acc); }
        else if (e - s <= SMALL_ROW || e - s > LONG_ROW) store_row<W, HINTS>(Y + j * W, acc, strm);
#pragma unroll
        for (int u = 0; u < 4; u++) k[u] = kn[u];
        s = s1; e = e1; s1 = s2; e1 = e2;
    }
}

// 8 lanes per list entry (a mid row, or one LONG_ROW-entry segment of a long row); entries sorted by length, descending.
// Three-stage software pipeline: list entry two steps ahead, col_idx batch one step ahead, gathers now.  Step t of group g
// handles list entry t * ngroups + g on even steps and t * ngroups + (ngroups - 1 - g) on odd ones, which evens out the totals per
// group.  The 8 lanes cover VG vertices x SPLIT record parts per unroll step.  ACC (union hops): a mid row is ORed into the stored
// record instead of replacing it (long-row segments merge with RED.OR either way).
template <int W, bool HINTS, int U, bool EARLY, bool ACC>
__global__ void __launch_bounds__(256)
k_pull_seg(const u32 *__restrict__ s_row, const u64 *__restrict__ s_start, const u32 *__restrict__ s_len, u64 ns,
           const u32 *__restrict__ ATj, const u64 *__restrict__ X, u64 *__restrict__ Y, const u64 *__restrict__ Gp,
           PullHints ph) {
    constexpr int WL = PullCfg<W>::WL, SPLIT = PullCfg<W>::SPLIT, VG = PullCfg<W>::VG;
    const u32 lane8 = threadIdx.x & 7;
    const u32 sub = (threadIdx.x & 31) >> 3;
    const u32 gmask = 0xFFu << (8 * sub);
    const u32 vi = lane8 / SPLIT, h = lane8 % SPLIT;
    const u64 *Xh = X + h * WL;
    const u64 keep = HINTS ? ph.gather_policy(X) : 0, strm = HINTS ? ph.stream_policy() : 0;
    u64 G[WL];
#pragma unroll
    for (int w = 0; w < WL; w++) G[w] = (EARLY && Gp) ? Gp[h * WL + w] : ~0ULL;
    const u64 ngroups = ((u64)gridDim.x * blockDim.x) >> 3;
    const u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 steps = (ns + ngroups - 1) / ngroups;
    auto entry = [&](u64 t) -> u64 { return t * ngroups + ((t & 1) ? ngroups - 1 - g : g); };
    auto fetch = [&](u64 t, u64 &s, u64 &e) {
        s = 0; e = 0;
        if (t < steps) {
            u64 i = entry(t);
            if (i < ns) {   // each entry is fetched once: with hints its lines skip L1
                s = HINTS ? ld_nc_once_u64(s_start + i, strm) : s_start[i];
                e = s + ((HINTS ? ld_nc_once_u32(s_len + i, strm) : s_len[i]) & ~SEG_ATOMIC);
            }
        }
    };
    u64 s0, e0, s1, e1;
    fetch(0, s0, e0);
    fetch(1, s1, e1);
    u32 k[U];
#pragma unroll
    for (int u = 0; u < U; u++) { u64 q = s0 + vi + VG * u; k[u] = (q < e0) ? ld_col<HINTS>(ATj + q, strm) : 0xFFFFFFFFu; }
    for (u64 t = 0; t < steps; t++) {
        u64 s2, e2;
        fetch(t + 2, s2, e2);
        u64 acc[WL];
#pragma unroll
        for (int w = 0; w < WL; w++) acc[w] = 0;
        u64 qb = s0;
        u32 it = 0;
        while (true) {
            const bool more = qb + VG * U < e0;
            const u64 nb = more ? qb + VG * U : s1, ne = more ? e0 : e1;
            u32 kn[U];
#pragma unroll
            for (int u = 0; u < U; u++) { u64 q = nb + vi + VG * u; kn[u] = (q < ne) ? ld_col<HINTS>(ATj + q, strm) : 0xFFFFFFFFu; }
#pragma unroll
            for (int u = 0; u < U; u++)
                if (k[u] != 0xFFFFFFFFu) or_words<WL, HINTS>(acc, Xh + (u64)k[u] * W, keep);
#pragma unroll
            for (int u = 0; u < U; u++) k[u] = kn[u];
            if (!more) break;
            if (EARLY) {   // stop once the entry holds the OR monoid's terminal value: cheap per-lane test, exact cross-lane OR every 4th
                bool full = true;
                if ((it & 3) == 3) {
#pragma unroll
                    for (int w = 0; w < WL; w++) {
                        u64 a = acc[w];
#pragma unroll
                        for (int d = SPLIT; d < 8; d <<= 1) a |= __shfl_xor_sync(gmask, a, d);
                        acc[w] = a;
                        full = full && (a == G[w]);
                    }
                } else {
#pragma unroll
                    for (int w = 0; w < WL; w++) full = full && (acc[w] == G[w]);
                }
                full = __all_sync(gmask, full);
                if (full) {
#pragma unroll
                    for (int u = 0; u < U; u++) { u64 q = s1 + vi + VG * u; k[u] = (q < e1) ? ld_col<HINTS>(ATj + q, strm) : 0xFFFFFFFFu; }
                    break;
                }
            }
            qb += VG * U;
            it++;
        }
#pragma unroll
        for (int w = 0; w < WL; w++) {
            u64 a = acc[w];
#pragma unroll
            for (int d = SPLIT; d < 8; d <<= 1) a |= __shfl_xor_sync(gmask, a, d);
            acc[w] = a;
        }
        if (e0 > s0 && vi == 0) {
            const u64 i = entry(t);
            u64 *dst = Y + (u64)(HINTS ? ld_nc_once_u32(s_row + i, strm) : s_row[i]) * W + h * WL;
            if ((HINTS ? ld_nc_once_u32(s_len + i, strm) : s_len[i]) & SEG_ATOMIC) {
#pragma unroll
                for (int w = 0; w < WL; w++) if (acc[w]) atomicOr((unsigned long long *)(dst + w), acc[w]);
            } else if (ACC) or_part<WL>(dst, acc);
            else store_part<WL, HINTS>(dst, acc, strm);
        }
        s0 = s1; e0 = e1; s1 = s2; e1 = e2;
    }
}

// ---- hot-set packing of the gather index space ------------------------------------------------------------------
// The pull gathers X[k] with k distributed like the out-degree of k.  Relabel k -> slot, slots ordered by out-degree
// descending and restricted to vertices that have out-edges at all (sinks are never gathered): the hot part of the
// frontier words becomes contiguous (L1/L2 resident), and the gather footprint shrinks from 8*W*n to 8*W*n1 bytes.
// shuffle (measurement, hot_shuffle): vertices with out-edges in the order of a hash of their id instead, so the gather
// source has no hot prefix at all; sinks stay last either way
__global__ void k_degree_keys(const u64 *__restrict__ Ap, u64 n, u64 *__restrict__ keys, u64 *__restrict__ n1, bool shuffle) {
    u64 v = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 cnt = 0;
    for (; v < n; v += stride) {
        u64 d = Ap[v + 1] - Ap[v];
        if (d > 0xFFFFFFFEULL) d = 0xFFFFFFFEULL;
        u64 hi = 0xFFFFFFFFULL - d;
        if (shuffle && d) { u32 h = (u32)v * 0x9E3779B1u; h ^= h >> 15; h *= 0x85EBCA77u; h ^= h >> 13; hi = h >> 1; }
        keys[v] = (hi << 32) | v;   // ascending sort => degree descending, then vertex id ascending
        cnt += d != 0;
    }
    if (cnt) atomicAdd((unsigned long long *)n1, cnt);
}
__global__ void k_slots_from_keys(const u64 *__restrict__ keys, const u64 *__restrict__ Ap, u64 n, u64 n1, u32 *__restrict__ vert,
                                  u32 *__restrict__ slot, u32 *__restrict__ hdeg) {
    u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; s < n; s += stride) {
        u32 v = (u32)(keys[s] & 0xFFFFFFFFULL);
        if (s < n1) {
            const u64 d = Ap[v + 1] - Ap[v];
            vert[s] = v; slot[v] = (u32)s; hdeg[s] = d > 0xFFFFFFFEULL ? 0xFFFFFFFEu : (u32)d;
        } else slot[v] = 0xFFFFFFFFu;
    }
}
__global__ void k_full_order(const u64 *__restrict__ keys, u64 n, u32 *__restrict__ pvert, u32 *__restrict__ pperm) {
    u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; s < n; s += stride) { const u32 v = (u32)(keys[s] & 0xFFFFFFFFULL); pvert[s] = v; pperm[v] = (u32)s; }
}
__global__ void k_relabel_cols(const u32 *__restrict__ j, u64 nnz, const u32 *__restrict__ slot, u32 *__restrict__ jp) {
    u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; q < nnz; q += stride) jp[q] = slot[j[q]];
}
template <int W>
__global__ void k_pack_frontier(const u32 *__restrict__ vert, u64 n1, const u64 *__restrict__ X, u64 *__restrict__ Xp) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n1 * W; t += stride) {
        u64 s = t / W, w = t % W;
        Xp[t] = X[(u64)vert[s] * W + w];
    }
}

// pack + flops + edges + OR-of-everything in one pass over the frontier (fused_prep): the hot set holds every vertex with
// out-edges, so flops = sum popc(X[v]) * deg(v) and edges = sum [X[v] != 0] * deg(v) over it are the exact totals, and
// G[w] = OR of word column w is the terminal value the pull kernels vote against.  One thread per packed word.
template <int W>
__global__ void __launch_bounds__(256)
k_pack_flops(const u32 *__restrict__ vert, const u32 *__restrict__ hdeg, u64 n1, const u64 *__restrict__ X, u64 *__restrict__ Xp,
             u64 *__restrict__ st /* [0] flops [1] edges */, u64 *__restrict__ G) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    __shared__ u64 sG[W];
    if (threadIdx.x < W) sG[threadIdx.x] = 0;
    __syncthreads();
    const u32 lane = threadIdx.x & 31;
    const u32 gmask = (W >= 32) ? 0xffffffffu : (((1u << W) - 1u) << (lane / W * W));   // the W lanes of one vertex
    u64 fl = 0, ed = 0, g = 0;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x, total = n1 * W;
    for (u64 base = t - lane; base < total; base += stride) {       // warp-uniform trip count (ballot inside)
        const u64 tt = base + lane;
        u64 x = 0;
        u32 d = 0;
        if (tt < total) {
            const u64 s = tt / W, w = tt % W;
            x = X[(u64)vert[s] * W + w];
            d = hdeg[s];
            Xp[tt] = x;
        }
        const u32 nz = __ballot_sync(0xffffffffu, x != 0) & gmask;
        fl += (u64)__popcll(x) * d;
        if (nz && (lane % W) == 0) ed += d;
        g |= x;
    }
    // OR across the lanes that hold the same word column (lane % W), then one shared atomic per column and warp
#pragma unroll
    for (int o = W; o < 32; o <<= 1) g |= __shfl_xor_sync(0xffffffffu, g, o);
    if (lane < W && g) atomicOr((unsigned long long *)&sG[lane], g);
    u64 tf = Red(ts).Sum(fl);
    __syncthreads();
    u64 te = Red(ts).Sum(ed);
    if (threadIdx.x == 0) {
        if (tf) atomicAdd((unsigned long long *)&st[0], tf);
        if (te) atomicAdd((unsigned long long *)&st[1], te);
    }
    __syncthreads();
    if (threadIdx.x < W && sG[threadIdx.x]) atomicOr((unsigned long long *)&G[threadIdx.x], sG[threadIdx.x]);
}

// the same totals for a frontier that already IS in hot-set order (permuted form): nothing to gather, nothing to write
template <int W>
__global__ void __launch_bounds__(256)
k_ordered_flops(const u32 *__restrict__ hdeg, u64 n1, const u64 *__restrict__ Xp, u64 *__restrict__ st, u64 *__restrict__ G) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    __shared__ u64 sG[W];
    if (threadIdx.x < W) sG[threadIdx.x] = 0;
    __syncthreads();
    const u32 lane = threadIdx.x & 31;
    const u32 gmask = (W >= 32) ? 0xffffffffu : (((1u << W) - 1u) << (lane / W * W));
    u64 fl = 0, ed = 0, g = 0;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x, total = n1 * W;
    for (u64 base = t - lane; base < total; base += stride) {
        const u64 tt = base + lane;
        u64 x = 0;
        u32 d = 0;
        if (tt < total) { x = Xp[tt]; d = hdeg[tt / W]; }
        const u32 nz = __ballot_sync(0xffffffffu, x != 0) & gmask;
        fl += (u64)__popcll(x) * d;
        if (nz && (lane % W) == 0) ed += d;
        g |= x;
    }
#pragma unroll
    for (int o = W; o < 32; o <<= 1) g |= __shfl_xor_sync(0xffffffffu, g, o);
    if (lane < W && g) atomicOr((unsigned long long *)&sG[lane], g);
    u64 tf = Red(ts).Sum(fl);
    __syncthreads();
    u64 te = Red(ts).Sum(ed);
    if (threadIdx.x == 0) {
        if (tf) atomicAdd((unsigned long long *)&st[0], tf);
        if (te) atomicAdd((unsigned long long *)&st[1], te);
    }
    __syncthreads();
    if (threadIdx.x < W && sG[threadIdx.x]) atomicOr((unsigned long long *)&G[threadIdx.x], sG[threadIdx.x]);
}

static void build_hot_pack(const DevCSR &A, const DevCSR &AT, PullTables &pt) {
    u64 n = A.nrows;
    pt.vert.release(); pt.jp.release(); pt.ap.release(); pt.ap_sorted = false; pt.slot.release(); pt.hdeg.release(); pt.n1 = 0; pt.packed = false;
    if (n == 0 || AT.nnz == 0 || n >= 0xFFFFFFFFULL) return;
    DevBuf<u64> keys(n), cnt(1);
    cnt.zero();
    LAUNCH(k_degree_keys, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, n, keys.ptr, cnt.ptr, ctx().opt_hot_shuffle != 0);
    sort_keys_u64(keys.ptr, n, 64);
    u64 n1 = read_scalar(cnt.ptr);
    pt.n1 = n1;
    pt.vert.alloc(n1 ? n1 : 1);
    pt.slot.alloc(n);
    pt.hdeg.alloc(n1 ? n1 : 1);
    LAUNCH(k_slots_from_keys, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, keys.ptr, A.p.ptr, n, n1, pt.vert.ptr, pt.slot.ptr, pt.hdeg.ptr);
    // the order over ALL vertices (the sort already put the sinks last, by id): frontiers may be stored in it (permuted form)
    pt.pvert = std::make_shared<DevBuf<u32>>(n);
    pt.pperm = std::make_shared<DevBuf<u32>>(n);
    LAUNCH(k_full_order, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, keys.ptr, n, pt.pvert->ptr, pt.pperm->ptr);
    static std::atomic<u64> next_tag{1};
    pt.perm_tag = next_tag.fetch_add(1);
    pt.packed = true;
}

// The pull tables of one matrix, built once per immutable base (B200_Matrix_prepare, or the first hop that pulls): the hot-set order
// when hot_pack is on, A'.col_idx and A.col_idx relabelled to it, and the segment list.  Turning hot_pack on after the tables
// were built without it adds the order and both relabelled col_idx arrays.
static void build_pull_tables(const DevCSR &A, const DevCSR &AT, PullTables &pt) {
    if (!pt.packed && ctx().opt_hot_pack) build_hot_pack(A, AT, pt);
    if (pt.packed && !pt.jp.ptr) {
        pt.jp.alloc(AT.nnz);
        LAUNCH(k_relabel_cols, grid_for(AT.nnz, 256, (u64)ctx().num_sms * 32), 256, 0, AT.j.ptr, AT.nnz, pt.slot.ptr, pt.jp.ptr);
    }
    // the CSR push's operand: A.col_idx already in the order it writes Y (4 * nnz(A) bytes), so a pushed flop needs no
    // dependent pperm[col] read from a table larger than L2.  Only when perm_push can read it; turning perm_push on later adds
    // it at the next build (until then the push reads pperm[col])
    if (pt.packed && !pt.ap.ptr && ctx().opt_perm_push && A.nnz && A.nrows == A.ncols) {
        pt.ap.alloc(A.nnz);
        LAUNCH(k_relabel_cols, grid_for(A.nnz, 256, (u64)ctx().num_sms * 32), 256, 0, A.j.ptr, A.nnz, pt.pperm->ptr, pt.ap.ptr);
    }
    // its rows ascending by position, for the sliced push (csr_push_sliced): OR commutes and only the CSR push reads ap, so the
    // order inside a row changes no result.  Like ap itself, added at the next build when push_slices was off at the first
    if (pt.ap.ptr && !pt.ap_sorted && ctx().opt_push_slices != 0 && A.nnz <= 0x7fffffffULL) {
        sort_rows_u32(A.p.ptr, A.nrows, pt.ap.ptr, A.nnz);
        pt.ap_sorted = true;
    }
    if (!pt.built) {
        build_seg_list(AT, pt);
        pt.built = true;
    }
}

// k_pull_small over every row of A', then k_pull_seg over the segment list.  The segment kernel's grid is every CTA resident at
// once (occupancy x SMs) unless pull_grid overrides it: entries are dealt round-robin to 8-lane groups, so one full wave keeps all
// SMs busy to the end.
template <int W, bool HINTS, bool ACC>
static void launch_pull(const DevCSR &AT, const PullTables &pt, u64 m, const u32 *gj, const u64 *gx, u64 *Y, const u64 *Gp,
                        PullHints ph) {
    Context &cx = ctx();
    LAUNCH((k_pull_small<W, HINTS, ACC>), grid_for(m, 256, (u64)cx.num_sms * 32), 256, 0, AT.p.ptr, gj, m, gx, Y, ph);
    if (!pt.ns) return;
    auto seg = [&](auto kern) {
        int per_sm = 0;
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, 0));
        if (per_sm < 1) per_sm = 1;
        if (cx.opt_pull_grid > 0) per_sm = (int)cx.opt_pull_grid;
        LAUNCH(kern, (u32)cx.num_sms * (u32)per_sm, 256, 0, pt.s_row.ptr, pt.s_start.ptr, pt.s_len.ptr, pt.ns, gj, gx, Y, Gp, ph);
    };
    if (Gp) seg(k_pull_seg<W, HINTS, 4, true, ACC>);
    else seg(k_pull_seg<W, HINTS, 4, false, ACC>);
}

// The pull's L2 policies, as measured on the H100 (scripts/pull_l2.py, DESIGN §4.8): from W = 2 up, the first half of the L2 of
// the gather source is evict_last and the rest evict_first (0.41 ms off a 4.6 ms W = 8 pull); the streams are evict_first only at
// W = 2 and 4, where that gains another 0.08 ms -- at W = 8 and 16 it costs 0.07-0.16 ms.  At W = 1 no policy pays.
// The prefix never exceeds the source.  (createpolicy.range takes 32-bit sizes: a source past 4 GB has its first 4 GB in the range.)
static bool pull_hints_on(int W) { const i64 o = ctx().opt_hints; return o > 0 || (o < 0 && W >= 2); }
static PullHints pull_hints(int W, u64 x_bytes) {
    const Context &cx = ctx();
    PullHints ph;
    ph.tot = x_bytes > 0xFFFFFFF0ULL ? 0xFFFFFFF0u : (u32)x_bytes;
    const u64 hot = cx.opt_hot_bytes >= 0 ? (u64)cx.opt_hot_bytes : cx.l2_bytes / 2;
    ph.hot = hot < ph.tot ? (u32)hot : ph.tot;
    ph.streams = cx.opt_hint_streams >= 0 ? cx.opt_hint_streams != 0 : (W == 2 || W == 4);
    return ph;
}

template <int W>
static void hop_impl(const DevBits &Xin, const DevCSR &A, const DevCSR *AT, PullTables *pt, DevBits &Y,
                     u64 *flops_out, int *path_out, bool acc) {
    Context &cx = ctx();
    u64 n = A.nrows, m = A.ncols;
    // X in permuted form: usable as it stands only by the pull through the tables it was ordered for; anything else works on a
    // natural-order copy (cannot happen on the bench path: the caller orders a frontier only for the operand it is pushed through)
    DevBits Xnat;
    const bool ordered = Xin.permuted() && AT && pt && pt->packed && Xin.perm_tag == pt->perm_tag && pt->jp.ptr && pt->hdeg.ptr &&
                         cx.opt_pull_mode != 0 && cx.opt_hot_pack && n == m;
    const DevBits *Xuse = &Xin;
    if (Xin.permuted() && !ordered) { bits_copy(Xin, Xnat); bits_naturalise(Xnat); Xuse = &Xnat; }
    const DevBits &X = *Xuse;
    if (!acc) {
        Y.clear();
        Y.nrows = X.nrows; Y.ncols = m; Y.W = W;
        Y.w.alloc(m * W);
    }
    DevBuf<u32> flag(n + 1);
    DevBuf<u64> st(2);
    st.zero();
    // fused_prep: when the hot-set tables exist, one pass packs the frontier for the pull AND yields flops / edges / the OR
    // terminal; the separate flops pass (needed for its per-vertex flags) then only runs if the push direction wins
    const bool fused = cx.opt_fused_prep && AT && pt && cx.opt_hot_pack && pt->packed && pt->jp.ptr && pt->hdeg.ptr &&
                       cx.opt_pull_mode != 0 && n == m;
    DevBuf<u64> Xp, Gd;
    if (ordered) {            // already in gather order: totals only
        Gd.alloc(W);
        Gd.zero();
        if (pt->n1) LAUNCH((k_ordered_flops<W>), grid_for(pt->n1 * W, 256, (u64)ctx().num_sms * 16), 256, 0, pt->hdeg.ptr, pt->n1, X.w.ptr, st.ptr, Gd.ptr);
    } else if (fused) {
        Xp.alloc(pt->n1 * W);
        Gd.alloc(W);
        Gd.zero();
        if (pt->n1) LAUNCH((k_pack_flops<W>), grid_for(pt->n1 * W, 256, (u64)ctx().num_sms * 16), 256, 0, pt->vert.ptr, pt->hdeg.ptr, pt->n1, X.w.ptr, Xp.ptr, st.ptr, Gd.ptr);
    } else if (n) LAUNCH(k_bits_flops, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, X.w.ptr, (u32)W, n, A.p.ptr, flag.ptr, st.ptr);
    u64 hst[2] = {0, 0};
    d2h(hst, st.ptr, 2);
    sync_stream();
    if (flops_out) *flops_out = hst[0];
    u64 edges = hst[1];
    bool pull = false;
    if (AT && pt) {
        if (cx.opt_pull_mode == 1) pull = true;
        else if (cx.opt_pull_mode == 0) pull = false;
        else pull = edges * 4 > A.nnz; // direction switch: frontier touches > 1/4 of the edges
    }
    if (edges == 0) { if (!acc) Y.w.zero(); if (path_out) *path_out = 0; return; }
    if (ordered && !pull) {                     // the push direction works on natural order: undo the frontier's order and start over
        DevBits Xn;
        bits_copy(Xin, Xn);
        bits_naturalise(Xn);
        hop_impl<W>(Xn, A, AT, pt, Y, flops_out, path_out, acc);
        return;
    }
    if (!pull) {
        if (fused) {                            // push needs the per-vertex active flags of the classic pass
            DevBuf<u64> st2(2);
            st2.zero();
            LAUNCH(k_bits_flops, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, X.w.ptr, (u32)W, n, A.p.ptr, flag.ptr, st2.ptr);
        }
        if (!acc) Y.w.zero();                   // accumulate: the REDs OR into the earlier operands' product
        CUDA_TRY(cudaMemsetAsync(flag.ptr + n, 0, sizeof(u32), stream()));
        DevBuf<u64> pos(n + 1);
        exclusive_scan_u32_to_u64(flag.ptr, pos.ptr, n + 1);
        u64 nact = read_scalar(pos.ptr + n);
        DevBuf<u32> act(nact);
        DevBuf<u64> cum(nact + 1), astart(nact);
        LAUNCH(k_compact_active, grid_for(n, 256, 1 << 16), 256, 0, flag.ptr, pos.ptr, n, A.p.ptr, act.ptr, cum.ptr, astart.ptr);
        CUDA_TRY(cudaMemsetAsync(cum.ptr + nact, 0, sizeof(u64), stream()));
        exclusive_scan_u64(cum.ptr, cum.ptr, nact + 1);
        u64 nchunks = (edges + PUSH_CHUNK - 1) / PUSH_CHUNK;
        {
            // col_idx segments + per-active (id,cum,start) + X words + one RED per (edge, word); the same bytes when accumulating
            TimedScope ts(acc ? TK_BITS_PUSH_ACC : TK_BITS_PUSH, 4 * edges + 20 * nact + 8ULL * W * nact + 8ULL * W * edges);
            LAUNCH((k_bits_push<W>), (u32)nchunks, 256, 0, act.ptr, cum.ptr, astart.ptr, nact, edges, A.j.ptr, X.w.ptr, Y.w.ptr);
        }
        if (path_out) *path_out = 2;
        return;
    }
    build_pull_tables(A, *AT, *pt);             // a no-op once the matrix has them
    const u32 *gj = AT->j.ptr;                  // gather index stream
    const u64 *gx = X.w.ptr;                    // gather source
    u64 gn = n;                                 // gather footprint in vertices
    if (ordered) {                              // the frontier already is the packed gather source (its first n1 records)
        gj = pt->jp.ptr; gx = X.w.ptr; gn = pt->n1;
    } else if (cx.opt_hot_pack && pt->packed) {
        if (!fused) {
            Xp.alloc(pt->n1 * W);
            if (pt->n1) LAUNCH((k_pack_frontier<W>), grid_for(pt->n1 * W, 256, (u64)ctx().num_sms * 32), 256, 0, pt->vert.ptr, pt->n1, X.w.ptr, Xp.ptr);
        }
        gj = pt->jp.ptr; gx = Xp.ptr; gn = pt->n1;
    }
    const u64 *Gp = nullptr;
    // opt_early_exit: 0 never, 1 auto, 2 always.  Auto: the in-loop vote pays for itself at W = 2 and 4 (hub rows saturate),
    // costs more than it saves at W = 1 (few rows ever hold all 64 bits) and at W >= 8; very dense frontiers always benefit.
    const bool dense_frontier = hst[0] >= (hst[1] * X.nrows) / 4;   // flops/edges = degree-weighted mean popcount of a gathered word
    if (cx.opt_early_exit == 2 || (cx.opt_early_exit == 1 && (dense_frontier || W == 2 || W == 4))) {
        if (!((fused && gx == Xp.ptr) || ordered)) {   // the fused / ordered pass already left the OR of the packed frontier in Gd
            Gd.alloc(W);
            Gd.zero();
            if (gn) LAUNCH((k_or_all<W>), grid_for(gn, 256, (u64)ctx().num_sms * 8), 256, 0, gx, gn, Gd.ptr);
        }
        Gp = Gd.ptr;
    }
    {
        // compulsory traffic: stream A' col_idx + rowptr, read X once, write Y once (X gathers hit L2).  Accumulating ("bits_pull_acc"),
        // Y is also read once: an upper bound, rows with nothing to add skip the read and the write.
        TimedScope ts(acc ? TK_BITS_PULL_ACC : TK_BITS_PULL, 4 * AT->nnz + 8 * (m + 1) + 8ULL * W * gn + (acc ? 16ULL : 8ULL) * W * m);
        const PullHints ph = pull_hints(W, gn * W * 8);
        const bool hints = pull_hints_on(W);
        if (acc) {
            if (hints) launch_pull<W, true, true>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
            else launch_pull<W, false, true>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
        } else if (hints) launch_pull<W, true, false>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
        else launch_pull<W, false, false>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
    }
    if (path_out) *path_out = 3;
}

// builds the pull tables of a square operand now (B200_Matrix_prepare) instead of inside the first hop that pulls
void bits_prepare_pull(const DevCSR &A, const DevCSR &AT, PullTables &pt) {
    if (A.nrows != A.ncols || !AT.nnz) return;
    build_pull_tables(A, AT, pt);
}

void bits_hop(const DevBits &X, const DevCSR &A, const DevCSR *AT, PullTables *pt, DevBits &Y, u64 *flops_out,
              int *path_out, bool acc) {
    if (X.ncols != A.nrows) throw GrbError(-6, "mxm: inner dimensions differ");
    if (acc) require_acc_target(Y, X.nrows, A.ncols, X.W);
    switch (X.W) {
    case 1: hop_impl<1>(X, A, AT, pt, Y, flops_out, path_out, acc); break;
    case 2: hop_impl<2>(X, A, AT, pt, Y, flops_out, path_out, acc); break;
    case 4: hop_impl<4>(X, A, AT, pt, Y, flops_out, path_out, acc); break;
    case 8: hop_impl<8>(X, A, AT, pt, Y, flops_out, path_out, acc); break;
    case 16: hop_impl<16>(X, A, AT, pt, Y, flops_out, path_out, acc); break;
    default: throw GrbError(-8, "bit-frontier: unsupported word count");
    }
}

// ---------------------------------------------------------------------------- elementwise
__global__ void k_bits_andnot(u64 *__restrict__ y, const u64 *__restrict__ m, u64 n) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) y[t] &= ~m[t];
}
__global__ void k_bits_or(u64 *__restrict__ y, const u64 *__restrict__ z, u64 n) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) y[t] |= z[t];
}
void bits_andnot(DevBits &Y, const DevBits &M) {
    require_natural(Y, "bits_andnot"); require_natural(M, "bits_andnot");
    if (Y.W != M.W || Y.ncols != M.ncols) throw GrbError(-6, "bits_andnot: shape mismatch");
    u64 n = Y.ncols * Y.W;
    if (n) LAUNCH(k_bits_andnot, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, Y.w.ptr, M.w.ptr, n);
}
void bits_or(DevBits &Y, const DevBits &Z) {
    require_natural(Y, "bits_or"); require_natural(Z, "bits_or");
    if (Y.W != Z.W || Y.ncols != Z.ncols) throw GrbError(-6, "bits_or: shape mismatch");
    u64 n = Y.ncols * Y.W;
    if (n) LAUNCH(k_bits_or, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, Y.w.ptr, Z.w.ptr, n);
}
void bits_copy(const DevBits &X, DevBits &Y) {
    Y.clear();
    Y.nrows = X.nrows; Y.ncols = X.ncols; Y.W = X.W;
    Y.w.alloc(X.ncols * X.W);
    d2d(Y.w.ptr, X.w.ptr, X.ncols * X.W);
    Y.pvert = X.pvert; Y.pperm = X.pperm; Y.perm_tag = X.perm_tag;       // a copy keeps the vertex order of its source
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
    if (threadIdx.x == 0) s_r0 = find_le64(Dp, 0, nrows - 1, lo);          // the two bounds are independent searches
    if (threadIdx.x == 32) s_r1 = find_le64(Dp, 0, nrows - 1, hi - 1);
    __syncthreads();
    const u64 r1 = s_r1;
    u64 k = s_r0;
    const u32 h = threadIdx.x % SPLIT;
    u64 fl = 0;
    for (u64 q = lo + threadIdx.x / SPLIT; q < hi; q += EPS) {
        k = find_le64(Dp, k, r1, q);                 // entries only move forward: the previous row bounds the search
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
    const u32 *xperm = X.permuted() ? X.pperm->ptr : nullptr, *yperm = Y.permuted() ? Y.pperm->ptr : nullptr;
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
    LAUNCH(k_csr_entry_info, grid_for(F.nrows * 32, 256), 256, 0, F.p.ptr, F.j.ptr, F.nrows, D.p.ptr, erow.ptr, cum.ptr,
           (u32 *)nullptr, (u64 *)nullptr);
    CUDA_TRY(cudaMemsetAsync(cum.ptr + F.nnz, 0, sizeof(u64), stream()));
    exclusive_scan_u64(cum.ptr, cum.ptr, F.nnz + 1);
    const u64 flops = read_scalar(cum.ptr + F.nnz);
    if (!flops) return 0;
    const u32 *yperm = Y.permuted() ? Y.pperm->ptr : nullptr;
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
    if ((Y.permuted() && !Y.pperm) || (Xb && Xb->permuted() && !Xb->pperm))
        throw GrbError(-101, "delta_lmxm: permuted frontier without its vertex -> position table");
    switch (Y.W) {
    case 1: return apply_deltas_impl<1>(Xb, Xc, dm, dp, Y);
    case 2: return apply_deltas_impl<2>(Xb, Xc, dm, dp, Y);
    case 4: return apply_deltas_impl<4>(Xb, Xc, dm, dp, Y);
    case 8: return apply_deltas_impl<8>(Xb, Xc, dm, dp, Y);
    case 16: return apply_deltas_impl<16>(Xb, Xc, dm, dp, Y);
    default: throw GrbError(-8, "bit-frontier: unsupported word count");
    }
}

// ---------------------------------------------------------------------------- exact dirty hop (reach over (m \ dm) u dp)
// delta_lmxm's AND-NOT term over-masks: it drops (i, j) whenever ANY deleted edge reaches j from row i, even when a remaining edge
// still reaches it.  A reach over a tensor with pending deletions needs X * (m \ dm) exactly.  Only the columns dm touches can
// differ from X * m, so those columns are recomputed: Y[pos(j)] = OR of X[pos(k)] over the in-edges k of m'(j, :) that are not in
// dm'(j, :).  Both rows are sorted, so a lane finds its in-edge in the deleted list with a lower bound that only moves forward.
// Hub columns are cut into REPAIR_SEG-entry segments, as the pull cuts long rows: a column of several segments is zeroed first and
// its segments arrive through RED.OR; a column of one segment is stored.  Work is O(W * the repaired columns' in-degrees).
static const u64 REPAIR_SEG = 1024;
static const u32 REPAIR_ATOMIC = 0x80000000u, REPAIR_FIRST = 0x40000000u, REPAIR_LEN = 0x3FFFFFFFu;

// segments per column: ceil(indeg_m(j) / REPAIR_SEG) where dm' has a row j, else 0;  st = {repaired columns, their in-edges}
__global__ void __launch_bounds__(256)
k_repair_count(const u64 *__restrict__ Dp, const u64 *__restrict__ Tp, u64 n, u32 *__restrict__ cnt, u64 *__restrict__ st) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 c = 0, e = 0;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j <= n; j += stride) {
        if (j == n) { cnt[j] = 0; continue; }
        const u64 d = Dp[j + 1] > Dp[j] ? Tp[j + 1] - Tp[j] : 0;
        cnt[j] = (u32)((d + REPAIR_SEG - 1) / REPAIR_SEG);
        c += d != 0;
        e += d;
    }
    const u64 tc = Red(ts).Sum(c);
    __syncthreads();
    const u64 te = Red(ts).Sum(e);
    if (threadIdx.x == 0) {
        if (tc) atomicAdd((unsigned long long *)&st[0], tc);
        if (te) atomicAdd((unsigned long long *)&st[1], te);
    }
}
__global__ void k_repair_emit(const u64 *__restrict__ Tp, const u32 *__restrict__ cnt, const u64 *__restrict__ pos, u64 n,
                              u32 *__restrict__ s_col, u64 *__restrict__ s_start, u32 *__restrict__ s_len) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const u32 c = cnt[j];
        if (!c) continue;
        const u64 t0 = Tp[j], d = Tp[j + 1] - t0, o = pos[j];
        for (u32 i = 0; i < c; i++) {
            const u64 s = (u64)i * REPAIR_SEG, len = d - s < REPAIR_SEG ? d - s : REPAIR_SEG;
            s_col[o + i] = (u32)j;
            s_start[o + i] = t0 + s;
            s_len[o + i] = (u32)len | (c > 1 ? (REPAIR_ATOMIC | (i == 0 ? REPAIR_FIRST : 0u)) : 0u);
        }
    }
}
// the columns merged with RED.OR start from zero (their first segment names them once)
template <int W>
__global__ void k_repair_zero(const u32 *__restrict__ s_col, const u32 *__restrict__ s_len, u64 ns, const u32 *__restrict__ yperm,
                              u64 *__restrict__ Y) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += stride) {
        if (!(s_len[i] & REPAIR_FIRST)) continue;
        const u64 j = s_col[i], py = yperm ? yperm[j] : j;
#pragma unroll
        for (int w = 0; w < W; w++) Y[py * W + w] = 0;
    }
}
// 8 lanes per segment, dealt round-robin; inside a group VG in-edges x SPLIT record parts per unroll step (the pull's lane split).
template <int W, int U>
__global__ void __launch_bounds__(256)
k_bits_repair(const u32 *__restrict__ s_col, const u64 *__restrict__ s_start, const u32 *__restrict__ s_len, u64 ns,
              const u32 *__restrict__ Tj, const u64 *__restrict__ Dp, const u32 *__restrict__ Dj, const u64 *__restrict__ X,
              const u32 *__restrict__ xperm, u64 *__restrict__ Y, const u32 *__restrict__ yperm) {
    constexpr int WL = PullCfg<W>::WL, SPLIT = PullCfg<W>::SPLIT, VG = PullCfg<W>::VG;
    const u32 lane8 = threadIdx.x & 7;
    const u32 gmask = 0xFFu << (8 * ((threadIdx.x & 31) >> 3));
    const u32 vi = lane8 / SPLIT, h = lane8 % SPLIT;
    const u64 *Xh = X + h * WL;
    const u64 ngroups = ((u64)gridDim.x * blockDim.x) >> 3;
    for (u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < ns; i += ngroups) {   // uniform inside the 8-lane group
        const u32 j = __ldg(s_col + i), fl = __ldg(s_len + i);
        const u64 s = __ldg(s_start + i), e = s + (fl & REPAIR_LEN), de = __ldg(Dp + j + 1);
        u64 d = __ldg(Dp + j);
        u64 acc[WL];
#pragma unroll
        for (int w = 0; w < WL; w++) acc[w] = 0;
        for (u64 qb = s; qb < e; qb += VG * U) {
            u32 k[U];
#pragma unroll
            for (int u = 0; u < U; u++) { const u64 q = qb + vi + VG * u; k[u] = q < e ? __ldg(Tj + q) : 0xFFFFFFFFu; }
#pragma unroll
            for (int u = 0; u < U; u++) {
                if (k[u] == 0xFFFFFFFFu) continue;
                u64 lo = d, hi = de;                 // lower bound of k[u] among the deleted sources of j
                while (lo < hi) {
                    const u64 mid = (lo + hi) >> 1;
                    if (__ldg(Dj + mid) < k[u]) lo = mid + 1; else hi = mid;
                }
                d = lo;
                if (d < de && __ldg(Dj + d) == k[u]) continue;   // a deleted edge
                const u64 px = xperm ? __ldg(xperm + k[u]) : k[u];
                or_words<WL, false>(acc, Xh + px * W, 0);
            }
        }
#pragma unroll
        for (int w = 0; w < WL; w++) {
            u64 a = acc[w];
#pragma unroll
            for (int dd = SPLIT; dd < 8; dd <<= 1) a |= __shfl_xor_sync(gmask, a, dd);
            acc[w] = a;
        }
        if (vi == 0) {
            const u64 py = yperm ? __ldg(yperm + j) : j;
            u64 *dst = Y + py * W + h * WL;
            if (fl & REPAIR_ATOMIC) {
#pragma unroll
                for (int w = 0; w < WL; w++) if (acc[w]) atomicOr((unsigned long long *)(dst + w), acc[w]);
            } else store_part<WL>(dst, acc);
        }
    }
}

void bits_repair_plan(const DevCSR &dm, const DevCSR &mT, RepairPlan &rp) {
    if (dm.nrows != mT.ncols || dm.ncols != mT.nrows) throw GrbError(-6, "reach: delta dimensions differ from the operand");
    rp.ns = rp.ncols = rp.inedges = 0;
    rp.s_col.release(); rp.s_len.release(); rp.s_start.release();
    rp.dmT.clear();
    const u64 n = mT.nrows;
    if (!dm.nnz || !n) return;
    transpose_csr(dm, rp.dmT, false);                  // dm changes with every write: built per call
    DevBuf<u32> cnt(n + 1);
    DevBuf<u64> pos(n + 1), st(2);
    st.zero();
    LAUNCH(k_repair_count, grid_for(n + 1, 256, (u64)ctx().num_sms * 16), 256, 0, rp.dmT.p.ptr, mT.p.ptr, n, cnt.ptr, st.ptr);
    exclusive_scan_u32_to_u64(cnt.ptr, pos.ptr, n + 1);
    u64 h[3];
    d2h(h, st.ptr, 2);
    d2h(h + 2, pos.ptr + n, 1);
    sync_stream();
    rp.ncols = h[0]; rp.inedges = h[1]; rp.ns = h[2];
    if (!rp.ns) return;
    rp.s_col.alloc(rp.ns); rp.s_len.alloc(rp.ns); rp.s_start.alloc(rp.ns);
    LAUNCH(k_repair_emit, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, mT.p.ptr, cnt.ptr, pos.ptr, n, rp.s_col.ptr,
           rp.s_start.ptr, rp.s_len.ptr);
}

template <int W>
static void repair_impl(const DevBits &X, const DevCSR &mT, const RepairPlan &rp, DevBits &Y) {
    const u32 *xperm = X.permuted() ? X.pperm->ptr : nullptr, *yperm = Y.permuted() ? Y.pperm->ptr : nullptr;
    // two row pointers per repaired column, m' and dm' column ids, the gathered records, the stored columns
    TimedScope ts(TK_BITS_REPAIR, 16 * rp.ncols + 4 * rp.inedges + 4 * rp.dmT.nnz + 8ULL * W * rp.inedges + 8ULL * W * rp.ncols);
    LAUNCH((k_repair_zero<W>), grid_for(rp.ns, 256, (u64)ctx().num_sms * 16), 256, 0, rp.s_col.ptr, rp.s_len.ptr, rp.ns, yperm, Y.w.ptr);
    static int per_sm = 0;
    if (!per_sm) {
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bits_repair<W, 4>, 256, 0));
        if (per_sm < 1) per_sm = 1;
    }
    const u64 need = (rp.ns * 8 + 255) / 256, full = (u64)ctx().num_sms * (u64)per_sm;
    LAUNCH((k_bits_repair<W, 4>), (u32)(need < full ? need : full), 256, 0, rp.s_col.ptr, rp.s_start.ptr, rp.s_len.ptr, rp.ns, mT.j.ptr,
           rp.dmT.p.ptr, rp.dmT.j.ptr, X.w.ptr, xperm, Y.w.ptr, yperm);
}

void bits_repair(const DevBits &X, const DevCSR &mT, const RepairPlan &rp, DevBits &Y) {
    if (!rp.ns) return;
    if (X.ncols != mT.ncols || Y.ncols != mT.nrows) throw GrbError(-6, "reach: frontier dimensions differ from the operand");
    if (X.W != Y.W) throw GrbError(-101, "reach: frontier and product word counts differ");
    if ((Y.permuted() && !Y.pperm) || (X.permuted() && !X.pperm))
        throw GrbError(-101, "reach: permuted frontier without its vertex -> position table");
    switch (Y.W) {
    case 1: repair_impl<1>(X, mT, rp, Y); break;
    case 2: repair_impl<2>(X, mT, rp, Y); break;
    case 4: repair_impl<4>(X, mT, rp, Y); break;
    case 8: repair_impl<8>(X, mT, rp, Y); break;
    case 16: repair_impl<16>(X, mT, rp, Y); break;
    default: throw GrbError(-8, "bit-frontier: unsupported word count");
    }
}

} // namespace b200
