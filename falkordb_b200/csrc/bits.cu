// bits.cu -- the frontier bit-matrix's form: CSR <-> bit-matrix, the row-major export, popcount, un-permuting, the elementwise
// ops and the diagonal (label) filter.
#include "frontier.cuh"

namespace b200 {

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
        const u64 r = last_le(Ap, 0, nrows - 1, q);   // the row of entry q
        u32 col = Aj[q];
        atomicOr((unsigned long long *)&X[(u64)col * W + (r >> 6)], 1ULL << (r & 63));
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
    csr_shape(C, X.nrows, n);
    if (n == 0) { C.p.zero(); return; }
    u64 ntiles = (n + TILE_V - 1) / TILE_V;
    u64 ncnt = (u64)64 * W * ntiles;
    DevBuf<u32> tc(ncnt + 1);
    DevBuf<u64> off(ncnt + 1);
    {
        TimedScope ts(TK_BITS_COUNT, 8ULL * W * n);
        const u64 nwarps = ntiles * pull_split((int)W);
        const u32 g = (u32)((nwarps + 3) / 4);
        with_words(W, [&](auto w) { LAUNCH((k_bits_count_csa<w>), g, 128, 0, X.w.ptr, n, ntiles, tc.ptr); });
    }
    CUDA_TRY(cudaMemsetAsync(tc.ptr + ncnt, 0, sizeof(u32), stream()));
    exclusive_scan_u32_to_u64(tc.ptr, off.ptr, ncnt + 1);
    LAUNCH(k_bits_rowptr, grid_for(X.nrows + 1, 256), 256, 0, off.ptr, X.nrows, ntiles, C.p.ptr);
    u64 nnz = read_scalar(off.ptr + X.nrows * ntiles);
    C.nnz = nnz;
    C.j.alloc(nnz);
    if (nnz) {
        TimedScope ts(TK_BITS_FILL, 8ULL * W * n + 4 * nnz);
        with_words(W, [&](auto w) { launch_fill<w>(X, ntiles, off.ptr, C.j.ptr); });
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

} // namespace b200
