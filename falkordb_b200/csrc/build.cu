// build.cu -- COO -> CSR build (GxB_Matrix_build_Scalar / GrB_Matrix_build_UINT64,
// reference call sites graph/src/graph/graphblas/matrix.rs:1199,1297), CSR transpose
// (GrB_transpose, matrix.rs:658) and the synthetic RMAT generator for the benchmark inputs.
//
// Pipeline: pack (row<<32|col) keys -> radix sort (CUB) -> mark run heads -> scan -> scatter
// unique cols (+ first value of each run: dup = ANY keeps the first tuple in input order)
// -> rowptr by per-row lower_bound over the sorted keys.
#include "common.cuh"
#include "ops.cuh"

namespace b200 {

static const u64 INVALID_KEY = ~0ULL;

__global__ void k_pack_keys(const u64 *__restrict__ I, const u64 *__restrict__ J, u64 n, u64 nrows, u64 ncols,
                            u64 *__restrict__ keys, u32 *__restrict__ err) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        u64 i = I[t], j = J[t];
        if (i >= nrows || j >= ncols) { *err = 1; keys[t] = INVALID_KEY; }
        else keys[t] = (i << 32) | j;
    }
}

__global__ void k_mark_heads(const u64 *__restrict__ keys, u64 n, u32 *__restrict__ head) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        u64 k = keys[t];
        head[t] = (k != INVALID_KEY && (t == 0 || keys[t - 1] != k)) ? 1u : 0u;
    }
}

// vals_src: original value array indexed by perm[t] (perm == null: no values)
__global__ void k_scatter_unique(const u64 *__restrict__ keys, const u32 *__restrict__ head,
                                 const u64 *__restrict__ pos, u64 n, u32 *__restrict__ outj,
                                 const u64 *__restrict__ perm, const u64 *__restrict__ vals_src,
                                 u64 *__restrict__ outx) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        if (head[t]) {
            u64 d = pos[t];
            outj[d] = (u32)(keys[t] & 0xffffffffULL);
            if (outx) outx[d] = vals_src[perm[t]];
        }
    }
}

// p[r] = number of unique valid keys with row < r
__global__ void k_rowptr_from_keys(const u64 *__restrict__ keys, const u64 *__restrict__ pos,
                                   const u32 *__restrict__ head, u64 n, u64 nrows, u64 *__restrict__ p) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; r <= nrows; r += stride) {
        // r >= 2^32 cannot happen for device matrices (nrows < 2^32)
        const u64 lo = lb64(keys, r >= ((u64)1 << 32) ? n : 0, n, r << 32);
        u64 v;
        if (lo == n) v = n ? pos[n - 1] + head[n - 1] : 0;
        else v = pos[lo];
        p[r] = v;
    }
}

// sorted keys (ascending; INVALID_KEY entries at the end are dropped; duplicates collapse)
static void csr_from_sorted_keys(const u64 *keys, u64 n, u64 nrows, u64 ncols, const u64 *perm,
                                 const u64 *vals_src, DevCSR &out) {
    csr_shape(out, nrows, ncols);
    if (n == 0) { out.p.zero(); return; }
    DevBuf<u32> head(n);
    DevBuf<u64> pos(n);
    LAUNCH(k_mark_heads, grid_for(n, 256, 1 << 20), 256, 0, keys, n, head.ptr);
    exclusive_scan_u32_to_u64(head.ptr, pos.ptr, n);
    u64 last_pos = read_scalar(pos.ptr + (n - 1));
    u32 last_head = read_scalar(head.ptr + (n - 1));
    u64 m = last_pos + last_head;
    out.nnz = m;
    out.j.alloc(m);
    if (vals_src) out.x.alloc(m);
    LAUNCH(k_scatter_unique, grid_for(n, 256, 1 << 20), 256, 0, keys, head.ptr, pos.ptr, n, out.j.ptr, perm, vals_src,
           vals_src ? out.x.ptr : nullptr);
    LAUNCH(k_rowptr_from_keys, grid_for(nrows + 1, 256, 1 << 20), 256, 0, keys, pos.ptr, head.ptr, n, nrows, out.p.ptr);
}

static int key_bits(u64 nrows) {
    int b = 0;
    while (b < 32 && ((u64)1 << b) < nrows) b++;
    int e = 32 + b + 1;
    return e > 64 ? 64 : e;
}

void build_from_device_coo(const u64 *dI, const u64 *dJ, const u64 *dX, u64 n, u64 nrows, u64 ncols, DevCSR &out,
                           bool *index_error) {
    if (nrows >= ((u64)1 << 32) || ncols >= ((u64)1 << 32))
        throw GrbError(-8, "device build: dimensions >= 2^32 are host-only");
    *index_error = false;
    if (n == 0) { csr_from_sorted_keys(nullptr, 0, nrows, ncols, nullptr, nullptr, out); return; }
    DevBuf<u64> keys(n);
    DevBuf<u32> err(1);
    err.zero();
    LAUNCH(k_pack_keys, grid_for(n, 256, 1 << 20), 256, 0, dI, dJ, n, nrows, ncols, keys.ptr, err.ptr);
    if (read_scalar(err.ptr)) { *index_error = true; return; }
    if (dX) {
        // stable radix sort => within a run of duplicates the first tuple in input order leads
        DevBuf<u64> perm(n);
        iota_u64(perm.ptr, n);
        sort_pairs_u64(keys.ptr, perm.ptr, n, 64);
        csr_from_sorted_keys(keys.ptr, n, nrows, ncols, perm.ptr, dX, out);
    } else {
        sort_keys_u64(keys.ptr, n, 64);
        csr_from_sorted_keys(keys.ptr, n, nrows, ncols, nullptr, nullptr, out);
    }
}

// ---- bulk tensor build (GRAPH.BULK: src/commands/bulk_insert.rs:497 -> graph.rs:2062 -> Tensor::set_all_from_slices, -------
// tensor.rs:333-447, applied to an EMPTY tensor) ---------------------------------------------------------------------------------
// From n (src, dst, edge id) triples: the forward UINT64 matrix whose value is the pair's edge id, or the MULTI_EDGE sentinel
// when the pair has more than one edge, plus the (pair key, edge id) list of every edge of every multi-edge pair (what the
// reference stores in `me`).  Two stable radix sorts ((id), then (src << 32 | dst)) put each pair's ids in ascending order inside
// its run; one pass marks the runs longer than one; the CSR comes out of the same sorted keys as every other build.
static const u64 TENSOR_MULTI_EDGE = ~0ULL;        // tensor.rs:206
__global__ void k_bulk_mark(const u64 *__restrict__ keys, const u64 *__restrict__ ids, u64 n, u64 *__restrict__ xval,
                            u32 *__restrict__ multi) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        const u64 k = keys[t];
        const bool dup = (t > 0 && keys[t - 1] == k) || (t + 1 < n && keys[t + 1] == k);
        xval[t] = dup ? TENSOR_MULTI_EDGE : ids[t];
        multi[t] = dup ? 1u : 0u;
    }
}
__global__ void k_bulk_compact(const u64 *__restrict__ keys, const u64 *__restrict__ ids, const u32 *__restrict__ multi,
                               const u64 *__restrict__ pos, u64 n, u64 *__restrict__ mkeys, u64 *__restrict__ mids) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride)
        if (multi[t]) { const u64 d = pos[t]; mkeys[d] = keys[t]; mids[d] = ids[t]; }
}
void tensor_bulk_build(const u64 *dI, const u64 *dJ, const u64 *dID, u64 n, u64 nrows, u64 ncols, DevCSR &fwd, DevBuf<u64> &mkeys,
                       DevBuf<u64> &mids, u64 *nmulti, bool *index_error) {
    if (nrows >= ((u64)1 << 32) || ncols >= ((u64)1 << 32))
        throw GrbError(-8, "device build: dimensions >= 2^32 are host-only");
    *index_error = false;
    *nmulti = 0;
    if (n == 0) { csr_from_sorted_keys(nullptr, 0, nrows, ncols, nullptr, nullptr, fwd); return; }
    DevBuf<u64> keys(n), ids(n);
    DevBuf<u32> err(1);
    err.zero();
    LAUNCH(k_pack_keys, grid_for(n, 256, 1 << 20), 256, 0, dI, dJ, n, nrows, ncols, keys.ptr, err.ptr);
    if (read_scalar(err.ptr)) { *index_error = true; return; }
    d2d(ids.ptr, dID, n);
    sort_pairs_u64(ids.ptr, keys.ptr, n, 64);            // by edge id
    sort_pairs_u64(keys.ptr, ids.ptr, n, 64);            // stable by pair: ids stay ascending inside a pair's run
    DevBuf<u64> xval(n), iota(n), pos(n);
    DevBuf<u32> multi(n);
    LAUNCH(k_bulk_mark, grid_for(n, 256, 1 << 20), 256, 0, keys.ptr, ids.ptr, n, xval.ptr, multi.ptr);
    iota_u64(iota.ptr, n);
    csr_from_sorted_keys(keys.ptr, n, nrows, ncols, iota.ptr, xval.ptr, fwd);
    exclusive_scan_u32_to_u64(multi.ptr, pos.ptr, n);
    const u64 nm = read_scalar(pos.ptr + (n - 1)) + read_scalar(multi.ptr + (n - 1));
    *nmulti = nm;
    if (nm) {
        mkeys.alloc(nm);
        mids.alloc(nm);
        LAUNCH(k_bulk_compact, grid_for(n, 256, 1 << 20), 256, 0, keys.ptr, ids.ptr, multi.ptr, pos.ptr, n, mkeys.ptr, mids.ptr);
    }
}

// ---- transpose --------------------------------------------------------------------------------
__global__ void k_transpose_keys(const u64 *__restrict__ p, const u32 *__restrict__ j, u64 nrows,
                                 u64 *__restrict__ keys) {
    // one warp per row, lanes stride over the row's entries
    u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    u32 lane = threadIdx.x & 31;
    for (u64 r = warp; r < nrows; r += nwarps) {
        u64 s = p[r], e = p[r + 1];
        for (u64 q = s + lane; q < e; q += 32) keys[q] = ((u64)j[q] << 32) | r;
    }
}

void transpose_csr(const DevCSR &A, DevCSR &out, bool keep_values) {
    u64 n = A.nnz;
    if (n == 0) { csr_from_sorted_keys(nullptr, 0, A.ncols, A.nrows, nullptr, nullptr, out); return; }
    // SURVEY 8(d) bytes_transpose = 2 * (4 * nnz + 4 * (n + 1)) (+ 2 * 8 * nnz if valued); the radix sort inside moves more
    TimedScope ts(TK_TRANSPOSE, 2 * (4 * n + 8 * (A.nrows + 1)) + ((keep_values && A.has_values()) ? 16 * n : 0));
    DevBuf<u64> keys(n);
    LAUNCH(k_transpose_keys, grid_for(A.nrows * 32, 256, 1 << 16), 256, 0, A.p.ptr, A.j.ptr, A.nrows, keys.ptr);
    int eb = key_bits(A.ncols);
    if (keep_values && A.has_values()) {
        DevBuf<u64> perm(n);
        iota_u64(perm.ptr, n);
        sort_pairs_u64(keys.ptr, perm.ptr, n, eb);
        csr_from_sorted_keys(keys.ptr, n, A.ncols, A.nrows, perm.ptr, A.x.ptr, out);
    } else {
        sort_keys_u64(keys.ptr, n, eb);
        csr_from_sorted_keys(keys.ptr, n, A.ncols, A.nrows, nullptr, nullptr, out);
    }
}

// ---- RMAT (identical stream to oracle/grb_oracle.c orc_rmat_edges) ------------------------------
__host__ __device__ inline u64 splitmix64(u64 x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
__device__ inline u64 scramble(u64 v, int scale, u64 k1, u64 k2) {
    u64 mask = ((u64)1 << scale) - 1;
    int sh = scale / 2 > 0 ? scale / 2 : 1;
    v = (v * k1) & mask;
    v ^= v >> sh;
    v = (v * k2) & mask;
    v ^= v >> sh;
    return v & mask;
}

// Row block [lo,hi) of the same RMAT matrix (by_col: row block of its transpose).  Every rank regenerates the global
// counter-based edge stream and keeps what it owns, so the union of the blocks is exactly rmat_csr's matrix.
__global__ void k_rmat_block_keys(int scale, u64 nedges, u64 seed, u64 k1, u64 k2, u64 lo, u64 hi, int by_col,
                                  u64 *__restrict__ keys) {
    const u32 TA = (u32)(0.57 * 4294967296.0), TB = (u32)((0.57 + 0.19) * 4294967296.0),
              TC = (u32)((0.57 + 0.19 + 0.19) * 4294967296.0);
    u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; e < nedges; e += stride) {
        u64 r = 0, c = 0, h = 0;
        for (int l = 0; l < scale; l++) {
            if ((l & 1) == 0) h = splitmix64(seed * 0xD1342543DE82EF95ULL + e * 64 + (u64)(l >> 1));
            u32 u = (l & 1) ? (u32)(h >> 32) : (u32)h;
            u32 rb, cb;
            if (u < TA) { rb = 0; cb = 0; } else if (u < TB) { rb = 0; cb = 1; }
            else if (u < TC) { rb = 1; cb = 0; } else { rb = 1; cb = 1; }
            r = (r << 1) | rb; c = (c << 1) | cb;
        }
        u64 i = scramble(r, scale, k1, k2), j = scramble(c, scale, k1, k2);
        if (by_col == 2) { u64 a = i > j ? i : j, c2 = i > j ? j : i; i = a; j = c2; }   // symmetrised lower triangle: (max, min)
        u64 own = by_col == 1 ? j : i, other = by_col == 1 ? i : j;
        keys[e] = (i == j || own < lo || own >= hi) ? INVALID_KEY : (((own - lo) << 32) | other);
    }
}

void rmat_block_csr(int scale, u64 edge_factor, u64 seed, u64 lo, u64 hi, int by_col, DevCSR &out) {
    if (scale < 1 || scale > 31) throw GrbError(-3, "rmat scale must be in [1,31]");
    u64 n = (u64)1 << scale, ne = n * edge_factor;
    if (lo > hi || hi > n) throw GrbError(-3, "rmat block out of range");
    u64 k1 = splitmix64(seed ^ 0xA5A5A5A5ULL) | 1ULL, k2 = splitmix64(seed ^ 0x5A5A5A5AULL) | 1ULL;
    DevBuf<u64> keys(ne);
    LAUNCH(k_rmat_block_keys, grid_for(ne, 256, 1 << 20), 256, 0, scale, ne, seed, k1, k2, lo, hi, by_col, keys.ptr);
    sort_keys_u64(keys.ptr, ne, 64);
    csr_from_sorted_keys(keys.ptr, ne, hi - lo, n, nullptr, nullptr, out);
}

void rmat_csr(int scale, u64 edge_factor, u64 seed, DevCSR &out) {
    if (scale < 1 || scale > 31) throw GrbError(-3, "rmat scale must be in [1,31]");
    rmat_block_csr(scale, edge_factor, seed, 0, (u64)1 << scale, 0, out);
}

} // namespace b200
