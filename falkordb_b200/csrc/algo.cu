// algo.cu -- the FP64 arithmetic corner of the path: GrB_mxv / GrB_vxm over GrB_PLUS_TIMES_SEMIRING_FP64 and
// GxB_PLUS_SECOND_FP64, and LAGr_PageRank built on it (graph/src/runtime/functions/algo_procedures.rs:744-752; LAGraph
// v1.x src/algorithm/LAGr_PageRank.c, not vendored -- restated in oracle/grb_oracle.c: orc_pagerank).
// Everything is HBM-bound streaming: one pass over the CSR (4 B col + 8 B value per entry) and a gather of x per entry.
// Summation order is FIXED (8 lanes per row, lane-strided partial sums, xor tree 4-2-1; block reductions over fixed chunks),
// so results repeat bit for bit from run to run and agree with the sequential oracle to ~1e-15 relative per term.
#include "common.cuh"
#include "ops.cuh"

namespace b200 {

// y[i] = (ACCUM ? y[i] : 0) + init + sum over row i of (VALUES ? a * x[k] : x[k]),  restricted to present x entries
template <bool VALUES>
__global__ void __launch_bounds__(256)
k_mxv_fp64(const u64 *__restrict__ p, const u32 *__restrict__ j, const u64 *__restrict__ ax, u64 nrows, const double *__restrict__ x,
           const unsigned char *__restrict__ present, double *__restrict__ y, unsigned char *__restrict__ ypresent, double init, int accum) {
    const u32 lane8 = threadIdx.x & 7, sub = (threadIdx.x & 31) >> 3;
    const u32 gmask = 0xFFu << (8 * sub);
    u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 ng = ((u64)gridDim.x * blockDim.x) >> 3;
    for (u64 base = g - sub; base < nrows; base += ng) {
        const u64 i = base + sub;
        if (i >= nrows) continue;
        const u64 s = p[i], e = p[i + 1];
        double acc = 0.0;
        bool any = false;
        for (u64 q = s + lane8; q < e; q += 8) {
            const u32 k = j[q];
            if (present && !present[k]) continue;
            acc += VALUES ? __longlong_as_double((long long)ax[q]) * x[k] : x[k];
            any = true;
        }
        acc += __shfl_xor_sync(gmask, acc, 4);
        acc += __shfl_xor_sync(gmask, acc, 2);
        acc += __shfl_xor_sync(gmask, acc, 1);
        any = __any_sync(gmask, any);
        if (lane8 == 0) {
            y[i] = (accum ? y[i] : 0.0) + init + acc;
            if (ypresent) ypresent[i] = any ? 1 : 0;
        }
    }
}
void mxv_fp64(const DevCSR &A, bool use_values, const double *x, const unsigned char *present, double *y, unsigned char *ypresent,
              double init, bool accum) {
    if (!A.nrows) return;
    // a valued matrix without entries has no value array on the device: its product is empty, not a domain error
    if (use_values && A.nnz && !A.has_values()) throw GrbError(-5, "PLUS_TIMES needs a valued matrix");
    // algorithmic bytes: col_idx + (values) + row pointers + one 8-byte gather per entry + y
    TimedScope ts(TK_MXV, (use_values ? 12 : 4) * A.nnz + 8 * (A.nrows + 1) + 8 * A.nnz + 8 * A.nrows);
    const u32 grid = grid_for(A.nrows * 8, 256, (u64)ctx().num_sms * 32);
    if (use_values) LAUNCH((k_mxv_fp64<true>), grid, 256, 0, A.p.ptr, A.j.ptr, A.x.ptr, A.nrows, x, present, y, ypresent, init, accum ? 1 : 0);
    else LAUNCH((k_mxv_fp64<false>), grid, 256, 0, A.p.ptr, A.j.ptr, (const u64 *)nullptr, A.nrows, x, present, y, ypresent, init, accum ? 1 : 0);
}

// ---- deterministic reductions: RED_BLOCKS fixed chunks, in-block strided partials + shared-memory tree, then one block ----
static const u32 RED_BLOCKS = 1024;
enum { RED_SINK = 0, RED_ABSDIFF = 1 };
template <int KIND>
__global__ void __launch_bounds__(256)
k_red_stage1(const double *__restrict__ a, const double *__restrict__ b, const u64 *__restrict__ Ap, u64 n, double *__restrict__ partial) {
    __shared__ double sh[256];
    const u64 chunk = (n + gridDim.x - 1) / gridDim.x;
    const u64 lo = (u64)blockIdx.x * chunk, hi = lo + chunk < n ? lo + chunk : n;
    double acc = 0.0;
    for (u64 i = lo + threadIdx.x; i < hi; i += 256) {
        if (KIND == RED_SINK) { if (Ap[i + 1] == Ap[i]) acc += a[i]; }
        else acc += fabs(a[i] - b[i]);
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (u32 s = 128; s; s >>= 1) { if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s]; __syncthreads(); }
    if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}
__global__ void __launch_bounds__(256) k_red_stage2(const double *__restrict__ partial, u32 m, double *__restrict__ out) {
    __shared__ double sh[256];
    double acc = 0.0;
    for (u32 i = threadIdx.x; i < m; i += 256) acc += partial[i];
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (u32 s = 128; s; s >>= 1) { if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s]; __syncthreads(); }
    if (threadIdx.x == 0) *out = sh[0];
}
__global__ void k_pr_init(const u64 *__restrict__ Ap, u64 n, double damping, double *__restrict__ d, double *__restrict__ r) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    const double dmin = 1.0 / damping, r0 = 1.0 / (double)n;
    for (; i < n; i += stride) {
        const double di = (double)(Ap[i + 1] - Ap[i]) / damping;
        d[i] = di > dmin ? di : dmin;
        r[i] = r0;
    }
}
__global__ void k_pr_scale(const double *__restrict__ r, const double *__restrict__ d, u64 n, double *__restrict__ t, double *__restrict__ w) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) { const double v = r[i]; t[i] = v; w[i] = v / d[i]; }
}

// A: adjacency pattern (out-degrees from its row pointers), AT: its transpose.  r: device double[n] (out).  Returns iterations.
int pagerank(const DevCSR &A, const DevCSR &AT, double damping, double tol, int itermax, double *r) {
    const u64 n = A.nrows;
    if (!n) return 0;
    DevBuf<double> t(n), w(n), d(n), partial(RED_BLOCKS), scal(2);
    const u32 g = grid_for(n, 256, (u64)ctx().num_sms * 16);
    LAUNCH(k_pr_init, g, 256, 0, A.p.ptr, n, damping, d.ptr, r);
    const double scaled = (1.0 - damping) / (double)n, damping_over_n = damping / (double)n;
    double rdiff = 1.0;
    int iters = 0;
    for (; iters < itermax && rdiff > tol; iters++) {
        LAUNCH((k_red_stage1<RED_SINK>), RED_BLOCKS, 256, 0, r, (const double *)nullptr, A.p.ptr, n, partial.ptr);
        LAUNCH(k_red_stage2, 1, 256, 0, partial.ptr, RED_BLOCKS, scal.ptr);
        double sink = 0.0;
        d2h(&sink, scal.ptr, 1);
        sync_stream();
        const double teleport = scaled + damping_over_n * sink;
        LAUNCH(k_pr_scale, g, 256, 0, r, d.ptr, n, t.ptr, w.ptr);
        mxv_fp64(AT, false, w.ptr, nullptr, r, nullptr, teleport, false);
        LAUNCH((k_red_stage1<RED_ABSDIFF>), RED_BLOCKS, 256, 0, t.ptr, r, A.p.ptr, n, partial.ptr);
        LAUNCH(k_red_stage2, 1, 256, 0, partial.ptr, RED_BLOCKS, scal.ptr + 1);
        d2h(&rdiff, scal.ptr + 1, 1);
        sync_stream();
    }
    return iters;
}


// ---- weakly connected components (algo.WCC -> LAGr_ConnectedComponents, algo_procedures.rs:838-846) ------------------------
// LAGraph's FastSV returns, for every vertex, the representative of its component; with min-hooking that is the smallest vertex id
// of the component, which is what this gives (deterministic).  A must have a symmetric pattern (the reference builds
// build_symmetric_adjacency_matrix and sets is_symmetric_structure).  Rounds of: hook every edge's larger root under the smaller
// (atomicMin), then full pointer jumping; O(log n) rounds, each one streaming pass over the CSR (4 B per entry + 8 B gathers).
__global__ void __launch_bounds__(256)
k_cc_hook(const u64 *__restrict__ p, const u32 *__restrict__ j, u64 n, u64 *__restrict__ parent, u32 *__restrict__ changed) {
    const u32 lane8 = threadIdx.x & 7;
    u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 ng = ((u64)gridDim.x * blockDim.x) >> 3;
    bool ch = false;
    for (u64 u = g; u < n; u += ng) {
        const u64 s = p[u], e = p[u + 1];
        if (s == e) continue;
        const u64 ru = parent[u];
        for (u64 q = s + lane8; q < e; q += 8) {
            const u64 rv = parent[j[q]];
            if (rv == ru) continue;
            const u64 hi = ru > rv ? ru : rv, lo = ru > rv ? rv : ru;
            atomicMin((unsigned long long *)&parent[hi], (unsigned long long)lo);
            ch = true;
        }
    }
    if (ch) *changed = 1;
}
__global__ void k_cc_jump(u64 *__restrict__ parent, u64 n) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        u64 r = parent[i];
        while (true) { const u64 rr = parent[r]; if (rr == r) break; r = rr; }
        parent[i] = r;
    }
}
int connected_components(const DevCSR &A, u64 *d_comp) {
    const u64 n = A.nrows;
    if (!n) return 0;
    const u32 g = grid_for(n, 256, (u64)ctx().num_sms * 16);
    iota_u64(d_comp, n);
    DevBuf<u32> changed(1);
    int rounds = 0;
    while (true) {
        changed.zero();
        LAUNCH(k_cc_hook, grid_for(n * 8, 256, (u64)ctx().num_sms * 32), 256, 0, A.p.ptr, A.j.ptr, n, d_comp, changed.ptr);
        LAUNCH(k_cc_jump, g, 256, 0, d_comp, n);
        rounds++;
        if (!read_scalar(changed.ptr)) break;
        if (rounds > 64) throw GrbError(-101, "connected components did not converge");
    }
    return rounds;
}

// ---- LAGraph_cdlp: community detection by synchronous label propagation (LDBC Graphalytics CDLP; algo_procedures.rs:1232) -------
// L0(v) = v; every round each vertex takes the most frequent label among its neighbours, the SMALLEST such label on ties; a vertex
// without neighbours keeps its label; stop after itermax rounds or at a fixed point.  One round = one key per entry
// (row << 32 | label of the neighbour), one radix sort over 32 + bits(n) bits -- the row field keeps every row's keys inside its
// own CSR segment [p[r], p[r+1]) -- and one pass that walks each sorted segment for its first longest run (ascending order makes
// the first longest run the minimum label).  8 B written + 8 B read per entry per pass; the sort's passes dominate.
__global__ void __launch_bounds__(256)
k_cdlp_keys(const u64 *__restrict__ p, const u32 *__restrict__ j, u64 n, const u64 *__restrict__ L, u64 *__restrict__ keys) {
    const u32 lane8 = threadIdx.x & 7;
    u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 ng = ((u64)gridDim.x * blockDim.x) >> 3;
    for (u64 u = g; u < n; u += ng) {
        const u64 s = p[u], e = p[u + 1];
        for (u64 q = s + lane8; q < e; q += 8) keys[q] = (u << 32) | L[j[q]];
    }
}
__global__ void __launch_bounds__(256)
k_cdlp_pick(const u64 *__restrict__ p, const u64 *__restrict__ keys, u64 n, const u64 *__restrict__ L, u64 *__restrict__ Lnew,
            u32 *__restrict__ changed) {
    u64 u = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    bool ch = false;
    for (; u < n; u += stride) {
        const u64 s = p[u], e = p[u + 1];
        u64 best = L[u];
        if (s < e) {
            u64 cur = keys[s] & 0xFFFFFFFFull, run = 1, best_run = 0;
            best = cur;
            for (u64 q = s + 1; q < e; ++q) {
                const u64 l = keys[q] & 0xFFFFFFFFull;
                if (l == cur) { ++run; continue; }
                if (run > best_run) { best_run = run; best = cur; }
                cur = l; run = 1;
            }
            if (run > best_run) best = cur;
        }
        Lnew[u] = best;
        ch |= best != L[u];
    }
    if (ch) *changed = 1;
}
int cdlp(const DevCSR &A, int itermax, u64 *d_label) {
    const u64 n = A.nrows;
    if (!n) return 0;
    if (n > (1ull << 32)) throw GrbError(-8, "cdlp: more than 2^32 vertices not supported");
    const u32 g = grid_for(n, 256, (u64)ctx().num_sms * 16);
    iota_u64(d_label, n);                                     // L0(v) = v
    if (!A.nnz) return 0;
    int bits_n = 1;
    while ((1ull << bits_n) < n) ++bits_n;
    DevBuf<u64> keys(A.nnz), next(n);
    DevBuf<u32> changed(1);
    u64 *cur = d_label, *nxt = next.ptr;
    int rounds = 0;
    for (; rounds < itermax; ) {
        changed.zero();
        LAUNCH(k_cdlp_keys, grid_for(n * 8, 256, (u64)ctx().num_sms * 32), 256, 0, A.p.ptr, A.j.ptr, n, cur, keys.ptr);
        sort_keys_u64(keys.ptr, A.nnz, 32 + bits_n);
        LAUNCH(k_cdlp_pick, g, 256, 0, A.p.ptr, keys.ptr, n, cur, nxt, changed.ptr);
        ++rounds;
        u64 *t = cur; cur = nxt; nxt = t;
        if (!read_scalar(changed.ptr)) break;
    }
    if (cur != d_label) CUDA_TRY(cudaMemcpyAsync(d_label, cur, n * sizeof(u64), cudaMemcpyDeviceToDevice, stream()));
    sync_stream();                                              // `next` is released on return
    return rounds;
}

} // namespace b200
