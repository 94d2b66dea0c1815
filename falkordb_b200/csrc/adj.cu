// adj.cu -- the induced effective layer of a relationship operand (B200_adjacency_delta, the adjacency the algorithm procedures run on).
// For one layer L (a base m with its pending deletes dm, or the pending inserts dp alone) and a monotone rank over the vertex ids,
// out(rank(v), rank(c)) for every entry (v, c) of L \ dm whose row and column are both kept.  Only the kept rows of L are read; a
// rank is monotone, so each output row is ascending as it is written.  Count pass, scan, fill pass, one warp per kept row; an entry
// is dropped when it sits in v's dm row, found by a forward-only search (each lane's columns only grow, so its cursor into the
// sorted dm row only moves forward).  The caller merges dp's layer in with ewise_union (dp wins over dm: its layer has no dm).
// Algorithmic bytes (kernel family "adj_build"): per kept row 16 B of row pointers for L and for dm, 4 B per column id of L and dm
// in those rows, 4 B of rank gather per column of L (kept-list form only), and the output: 4 B per entry + 8 B per row pointer.
#include "common.cuh"
#include "ops.cuh"

namespace b200 {

static constexpr u32 ADJ_DROP = 0xffffffffu;

// row(r) = the vertex output row r reads (>= n: none), rank(c) = c's output column or ADJ_DROP
struct RankIdentity {             // keep == NULL: rank(v) = v below n_out, dropped from n_out on (dup + resize)
    u64 n_out;
    __device__ __forceinline__ u64 row(u64 r) const { return r; }
    __device__ __forceinline__ u32 rank(u32 c) const { return c < n_out ? c : ADJ_DROP; }
};
struct RankTable {                // keep[r] = the r-th kept vertex, tab[v] = v's position in keep or ADJ_DROP
    const u64 *keep; const u32 *tab;
    __device__ __forceinline__ u64 row(u64 r) const { return keep[r]; }
    __device__ __forceinline__ u32 rank(u32 c) const { return tab[c]; }
};

// One warp walks row v of L in 32-entry strides; lane keeps its own cursor into v's dm row.  FILL: write the surviving entries'
// ranks from Cp[r] on (ballot prefix keeps them in order), else store the row's count.  in_rows (timing only): the L and dm
// entries of the kept rows.
template <class Rank, bool FILL>
__global__ void __launch_bounds__(256)
k_adj_layer(const u64 *__restrict__ Lp, const u32 *__restrict__ Lj, const u64 *__restrict__ Dp, const u32 *__restrict__ Dj,
            u64 n, u64 rows, Rank rk, u32 *__restrict__ cnt, const u64 *__restrict__ Cp, u32 *__restrict__ Cj,
            unsigned long long *__restrict__ in_rows) {
    const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u32 lane = threadIdx.x & 31, lt = (1u << lane) - 1u;
    u64 seen_l = 0, seen_d = 0;
    for (u64 r = warp; r < rows; r += nwarps) {
        const u64 v = rk.row(r);
        u64 s = 0, e = 0, ds = 0, de = 0;
        if (v < n) { s = Lp[v]; e = Lp[v + 1]; if (Dp) { ds = Dp[v]; de = Dp[v + 1]; } }
        seen_l += e - s;
        seen_d += de - ds;
        u64 o = FILL ? Cp[r] : 0;
        if (FILL && Cp[r + 1] == o) continue;
        u32 c = 0;
        u64 dq = ds;                                        // this lane's cursor into the dm row
        for (u64 q0 = s; q0 < e; q0 += 32) {
            const u64 q = q0 + lane;
            u32 out = ADJ_DROP;
            if (q < e) {
                const u32 col = Lj[q];
                out = rk.rank(col);
                if (out != ADJ_DROP && dq < de) {
                    dq = lb32(Dj, dq, de, col);
                    if (dq < de && Dj[dq] == col) out = ADJ_DROP;
                }
            }
            const u32 m = __ballot_sync(0xffffffffu, out != ADJ_DROP);
            if (FILL) {
                if (out != ADJ_DROP) Cj[o + __popc(m & lt)] = out;
                o += __popc(m);
            } else {
                c += __popc(m);
            }
        }
        if (!FILL && lane == 0) cnt[r] = c;
    }
    if (in_rows && lane == 0) {                            // timing runs only: one add per warp
        atomicAdd(&in_rows[0], (unsigned long long)seen_l);
        atomicAdd(&in_rows[1], (unsigned long long)seen_d);
    }
}

__global__ void k_adj_rank_scatter(const u64 *__restrict__ keep, u64 nkeep, u32 *__restrict__ tab) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < nkeep; t += stride) tab[keep[t]] = (u32)t;
}

void adj_rank_table(const u64 *d_keep, u64 nkeep, u64 n, DevBuf<u32> &tab) {
    tab.alloc(n ? n : 1);
    fill_u32(tab.ptr, ADJ_DROP, n);
    if (nkeep) LAUNCH(k_adj_rank_scatter, grid_for(nkeep, 256, (u64)ctx().num_sms * 16), 256, 0, d_keep, nkeep, tab.ptr);
}

template <class Rank>
static void adj_layer_run(const DevCSR &L, const DevCSR *dm, u64 rows, Rank rk, bool gather, DevCSR &out) {
    csr_shape(out, rows, rows);
    if (rows == 0 || L.nnz == 0) { out.p.zero(); return; }
    const u64 *Dp = dm && dm->nnz ? dm->p.ptr : nullptr;
    const u32 *Dj = Dp ? dm->j.ptr : nullptr;
    const bool timing = ctx().opt_timing != 0;
    DevBuf<unsigned long long> seen;
    if (timing) { seen.alloc(2); seen.zero(); }
    DevBuf<u32> cnt(rows + 1);
    const u32 grid = grid_for(rows * 32, 256, (u64)ctx().num_sms * 32);
    timed_begin(TK_ADJ_BUILD);
    LAUNCH((k_adj_layer<Rank, false>), grid, 256, 0, L.p.ptr, L.j.ptr, Dp, Dj, L.nrows, rows, rk, cnt.ptr, (const u64 *)nullptr,
           (u32 *)nullptr, timing ? seen.ptr : nullptr);
    const u64 nnz = csr_rows_from_counts(cnt.ptr, rows, out, false);
    if (nnz)
        LAUNCH((k_adj_layer<Rank, true>), grid, 256, 0, L.p.ptr, L.j.ptr, Dp, Dj, L.nrows, rows, rk, (u32 *)nullptr, out.p.ptr, out.j.ptr,
               (unsigned long long *)nullptr);
    u64 in[2] = {0, 0};
    if (timing) { d2h(in, (const u64 *)seen.ptr, 2); sync_stream(); }
    // the compulsory bytes: row pointers of L and dm for each kept row, their column ids in those rows (each entry once, the
    // count and fill passes both read them), a rank gather per column (kept-list form), the output once
    timed_end(TK_ADJ_BUILD, 16 * rows * (Dp ? 2 : 1) + 4 * (in[0] + in[1]) + (gather ? 4 * in[0] : 0) + 4 * nnz + 8 * (rows + 1));
}

void adj_layer(const DevCSR &L, const DevCSR *dm, u64 n_out, const u64 *d_keep, const u32 *rank_tab, u64 nkeep, DevCSR &out) {
    if (d_keep) adj_layer_run(L, dm, nkeep, RankTable{d_keep, rank_tab}, true, out);
    else adj_layer_run(L, dm, n_out, RankIdentity{n_out}, false, out);
}

} // namespace b200
