// common.cuh -- device-memory, stream, launch-accounting and error plumbing shared by every
// translation unit of libb200grb.so (the H100-native (sm_90a) GraphBLAS traversal backend).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include <stdexcept>
#include <string>
#include <vector>
#include <memory>
#include <cstdio>

namespace b200 {

typedef uint32_t u32;
typedef uint64_t u64;
typedef int64_t i64;

struct CudaError : std::runtime_error {
    cudaError_t code;
    CudaError(cudaError_t c, const char *file, int line)
        : std::runtime_error(std::string(cudaGetErrorName(c)) + ": " + cudaGetErrorString(c) + " at " + file + ":" +
                             std::to_string(line)),
          code(c) {}
};
struct GrbError : std::runtime_error {
    int info;
    GrbError(int i, const std::string &m) : std::runtime_error(m), info(i) {}
};

#define CUDA_TRY(expr)                                                    \
    do {                                                                  \
        cudaError_t e__ = (expr);                                         \
        if (e__ != cudaSuccess) throw ::b200::CudaError(e__, __FILE__, __LINE__); \
    } while (0)

// ---- global context (one process per GPU; one library stream) -------------------------------
struct Context {
    bool ready = false;
    int device = 0;
    int num_sms = 132;                // read from the device at bring-up (prims.cu)
    u64 l2_bytes = 50ULL << 20;       // likewise: the L2 cache the sliced CSR push sizes its destination slices by
    cudaStream_t stream = nullptr;
    std::atomic<u64> launches{0};     // kernels of THIS library launched (bench.py gpu_launches)
    std::atomic<u64> lib_launches{0}; // CUB primitives launched on our behalf (sort / scan)
    // last-op statistics (read through B200_get_stat)
    std::atomic<u64> last_flops{0}, total_flops{0}, last_path{0};
    std::atomic<u64> h2d_bytes{0}, d2h_bytes{0};
    // tunables (B200_set_option)
    i64 opt_bits_mode = -1;        // -1 auto, 0 never use the bit-frontier path, 1 always when legal
    i64 opt_pull_mode = -1;        // -1 auto, 0 push only, 1 pull only
    i64 opt_small_cap = 4096;      // rows with <= this many flops use the shared-memory sort path
    i64 opt_bitmap_budget = (i64)2 << 30; // bytes of global bitmap scratch per heavy-row wave
    i64 opt_bits_min_flops = 1 << 22;     // auto mode: use bit-frontier when flops >= this
    i64 opt_sync_after_op = 0;
    i64 opt_timing = 0;
    i64 opt_perm_push = 1;         // a CSR frontier pushed through a prepared matrix lands in that matrix's hot-set order (no packing pass before the next pull)
    i64 opt_bfs_direction = 0;     // 0 = direction-optimising, 1 = top-down only, 2 = bottom-up only (test hooks)
    i64 opt_bfs_sparse_exchange = 1;   // partitioned BFS: ship discovered-vertex lists instead of bitmaps when the frontier is sparse
    i64 opt_early_exit = 1;        // stop a pull row once it holds the OR monoid's terminal value (exact)
    i64 opt_hints = -1;            // L2 cache policies in the pull kernels: -1 = as measured (on for W >= 2; bits_hop.cu: pull_hints), 0 / 1 = off / on
    i64 opt_hint_streams = -1;     // with hints on, the pull's streams (A' col_idx and rowptr, segment list, Y) are evict_first: -1 = as measured (W = 2, 4), 0 / 1
    i64 opt_hot_bytes = -1;        // evict_last prefix of the pull's gather source: -1 = half of l2_bytes, 0 = the gathers are evict_normal
    i64 opt_hot_shuffle = 0;       // measurement: pull tables built from now on order their hot set by a hash, not by out-degree
    i64 opt_hot_pack = 1;          // gather through the degree-sorted, sink-free relabelling of the frontier
    i64 opt_fused_prep = 1;        // pull hops: pack the frontier, count flops / edges and OR it in one pass
    i64 opt_csr_push = 1;          // small CSR frontiers push straight from their entries (no O(n*W) bit-matrix passes); 2 = whatever their size (measurement)
    i64 opt_push_slices = -1;      // the CSR push through a prepared operand issues its REDs in L2-sized destination slices: -1 = slices sized from the L2, 0 = off (entry order), k > 0 = k slices (measurement and tests)
    i64 opt_diag_filter = 1;       // frontier-form mxm by a diagonal (label) matrix runs as an elementwise column filter
    i64 opt_pull_grid = 0;         // CTAs per SM of the segment pull kernel (0 = occupancy: one resident wave)
    i64 opt_union_accum = 1;       // union hops: clean extra operands OR into one product (0 = a product per operand plus an OR pass; measurement)
    i64 opt_shortest_path_budget = 0;   // B200_shortest_path / B200_all_shortest_paths: neighbour entries per piece of a round or level (0 = a sixteenth of free memory's worth)
};
Context &ctx();
void ensure_init();

inline cudaStream_t stream() { return ctx().stream; }

// ---- optional per-kernel timing (CUDA events on the launch stream; B200_set_option("timing",1)) ----
enum TimedId { TK_BITS_PULL = 0, TK_BITS_PUSH, TK_HEAVY_ACC, TK_SMALL_ROWS, TK_BITS_FILL, TK_BITS_COUNT,
               TK_BITMAP_EXPAND, TK_BFS_EXPAND, TK_UNION, TK_FILTER, TK_MXV, TK_MASKED, TK_TRANSPOSE, TK_BITS_DELTA,
               TK_BITS_REPAIR, TK_BITS_PULL_ACC, TK_BITS_PUSH_ACC, TK_EDGE_EXPAND, TK_BFS_DELTA, TK_ADJ_BUILD,
               TK_TENSOR_WRITE, TK_VAR_LEN_TRAILS, TK_VAR_LEN_REACH_BOTH, TK_SHORTEST_PATH, TK_ALL_SHORTEST_PATHS,
               TK_COUNT_ };
const char *timed_name(int id);
void timed_begin(int id);
void timed_end(int id, u64 algorithmic_bytes) noexcept;
struct TimedScope {
    int id; u64 bytes;
    TimedScope(int i, u64 b) : id(i), bytes(b) { timed_begin(id); }
    ~TimedScope() { timed_end(id, bytes); }
};
// drains recorded events: total ms / launches / bytes per id
void timed_collect(double *ms, u64 *launches, u64 *bytes);
void timed_reset();

// ---- caching device allocator (prims.cu) ----------------------------------------------------------
// Size-class free lists over cudaMalloc.  Every buffer is only ever touched by work enqueued on the one library
// stream, so a freed block can be handed out again immediately (stream order guarantees the previous user is done
// before the next one starts): steady state has no driver allocation calls and no pool growth / fragmentation.
void *pool_alloc(size_t bytes);
void pool_free(void *p);
void pool_trim();
size_t pool_bytes_cached();

// ---- device buffers -------------------------------------------------------------------------------
template <typename T>
struct DevBuf {
    T *ptr = nullptr;
    size_t n = 0;
    DevBuf() {}
    explicit DevBuf(size_t count) { alloc(count); }
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : ptr(o.ptr), n(o.n) { o.ptr = nullptr; o.n = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { release(); ptr = o.ptr; n = o.n; o.ptr = nullptr; o.n = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    void alloc(size_t count) {
        release();
        n = count;
        if (count == 0) { ptr = nullptr; return; }
        ptr = (T *)pool_alloc(count * sizeof(T));
    }
    void release() {
        if (ptr) { pool_free(ptr); ptr = nullptr; }
        n = 0;
    }
    void zero() { if (n) CUDA_TRY(cudaMemsetAsync(ptr, 0, n * sizeof(T), stream())); }
    T *release_ownership() { T *p = ptr; ptr = nullptr; n = 0; return p; }
    size_t bytes() const { return n * sizeof(T); }
};

// Small device-to-host reads (scalars the host steers by: flops, nnz, bin counts) do not use the copy engine: a one-warp
// kernel stores them into mapped pinned memory and sync_stream() hands them to their destinations.  A DMA read-back would
// queue behind whatever the D2H engine is busy with -- e.g. the 100+ MB result bitmap of the previous batch slice travelling
// on the copy stream -- and stall the compute stream for milliseconds (prims.cu).
bool small_read(void *dst, const void *src, size_t bytes);   // false: not taken (too large / no slot), use a memcpy
void flush_small_reads();                                    // after the stream has been synchronised
void drop_small_reads();                                     // error paths: pending deliveries are abandoned, not copied
inline void sync_stream() { CUDA_TRY(cudaStreamSynchronize(stream())); flush_small_reads(); }

template <typename T>
inline T read_scalar(const T *dptr) {
    T v;
    if (!small_read(&v, dptr, sizeof(T))) CUDA_TRY(cudaMemcpyAsync(&v, dptr, sizeof(T), cudaMemcpyDeviceToHost, stream()));
    sync_stream();
    return v;
}
template <typename T>
inline void h2d(T *dst, const T *src, size_t n) {
    if (n) { CUDA_TRY(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, stream())); ctx().h2d_bytes += n * sizeof(T); }
}
template <typename T>
inline void d2h(T *dst, const T *src, size_t n) {
    if (n) {
        if (!small_read(dst, src, n * sizeof(T))) CUDA_TRY(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToHost, stream()));
        ctx().d2h_bytes += n * sizeof(T);
    }
}
template <typename T>
inline void d2d(T *dst, const T *src, size_t n) {
    if (n) CUDA_TRY(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyDeviceToDevice, stream()));
}

// Kernel launch with accounting.  Usage: LAUNCH(kernel, grid, block, smem, args...)
#define LAUNCH(kern, grid, block, smem, ...)                                   \
    do {                                                                       \
        ::b200::ctx().launches.fetch_add(1, std::memory_order_relaxed);        \
        kern<<<(grid), (block), (smem), ::b200::stream()>>>(__VA_ARGS__);      \
        CUDA_TRY(cudaGetLastError());                                          \
    } while (0)

inline u32 grid_for(u64 items, u32 per_block, u64 cap = 0x7fffffffULL) {
    u64 g = (items + per_block - 1) / per_block;
    if (g < 1) g = 1;
    if (g > cap) g = cap;
    return (u32)g;
}

// ---- device CSR -----------------------------------------------------------------------------
// rowptr u64[nrows+1], col u32[nnz] ascending within a row, val u64[nnz] or null (iso/pattern).
struct DevCSR {
    u64 nrows = 0, ncols = 0, nnz = 0;
    DevBuf<u64> p;
    DevBuf<u32> j;
    DevBuf<u64> x; // empty => pattern-only (every stored value is true / 1)
    bool has_values() const { return x.ptr != nullptr; }
    void clear() { p.release(); j.release(); x.release(); nnz = 0; }
};

// frontier bit-matrix: an r x n boolean matrix (r <= 64*W) stored vertex-major:
// word[v*W + w] bit b  <=>  entry (row 64*w+b, col v).
struct DevBits {
    u64 nrows = 0, ncols = 0;
    u32 W = 0;
    DevBuf<u64> w;
    // Permuted form (bits_hop.cu, "hot-set order"): the words of vertex v live at position pos(v) instead of v, pos = the degree-sorted
    // gather order of the matrix this frontier is about to be multiplied by (PullTables::pperm), so the pull of the next hop gathers
    // straight from it with no packing pass.  pvert[position] = vertex undoes it; perm_tag names the permutation (0 = natural).
    // pperm[vertex] = position addresses single vertices in place (the delta terms of a dirty hop).
    std::shared_ptr<DevBuf<u32>> pvert, pperm;
    u64 perm_tag = 0;
    bool valid() const { return w.ptr != nullptr; }
    bool permuted() const { return perm_tag != 0; }
    void clear() { w.release(); W = 0; pvert.reset(); pperm.reset(); perm_tag = 0; }
};

// ---- L2 residency hints (createpolicy descriptors; sm_80+) ---------------------------------------
// keep  : data that is gathered at random and must stay L2-resident (the frontier bit-matrix X)
// stream: data read or written exactly once (col_idx / rowptr streams, outputs)
#ifdef __CUDACC__
__device__ __forceinline__ u64 policy_keep() { u64 p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 policy_stream() { u64 p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
// [base, base+primary) evict_last (kept resident), the rest of [base, base+total) evict_first: the hot prefix of the
// degree-sorted packed frontier stays in L2 while its cold tail streams through
__device__ __forceinline__ u64 policy_range(const void *base, u32 primary_bytes, u32 total_bytes) {
    u64 p;
    asm volatile("createpolicy.range.L2::evict_last.L2::evict_first.b64 %0, [%1], %2, %3;" : "=l"(p) : "l"(base), "r"(primary_bytes), "r"(total_bytes));
    return p;
}
__device__ __forceinline__ u64 policy_normal() { u64 p; asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p)); return p; }
// Read-only loads with an L2 policy.  They are non-volatile asm on the non-coherent path (ld.global.nc, what __ldg issues), so
// the compiler schedules them as freely as __ldg: a kernel's software pipeline keeps its loads in flight across each other.
// Only for data that nothing writes while the kernel runs.  _once: L1::no_allocate, for lines no later load of the thread reuses.
__device__ __forceinline__ ulonglong2 ld_nc_v2(const ulonglong2 *p, u64 pol) {
    ulonglong2 v;
    asm("ld.global.nc.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(v.x), "=l"(v.y) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ u64 ld_nc_u64(const u64 *p, u64 pol) {
    u64 v; asm("ld.global.nc.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ u32 ld_nc_u32(const u32 *p, u64 pol) {
    u32 v; asm("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ u64 ld_nc_once_u64(const u64 *p, u64 pol) {
    u64 v; asm("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ u32 ld_nc_once_u32(const u32 *p, u64 pol) {
    u32 v; asm("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ void st_v2_hint(ulonglong2 *p, ulonglong2 v, u64 pol) {
    asm volatile("st.global.L2::cache_hint.v2.u64 [%0], {%1, %2}, %3;" ::"l"(p), "l"(v.x), "l"(v.y), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_u64_stream(u64 *p, u64 v, u64 pol) {
    asm volatile("st.global.L2::cache_hint.u64 [%0], %1, %2;" ::"l"(p), "l"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_u32_stream(u32 *p, u32 v, u64 pol) {
    asm volatile("st.global.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(p), "r"(v), "l"(pol) : "memory");
}

// ---- searches over ascending arrays ----
// the first position in j[lo, hi) whose value is not below c
__device__ __forceinline__ u64 lb32(const u32 *__restrict__ j, u64 lo, u64 hi, u32 c) {
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (j[mid] < c) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ u64 lb64(const u64 *__restrict__ k, u64 lo, u64 hi, u64 key) {
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (k[mid] < key) lo = mid + 1; else hi = mid; }
    return lo;
}
// the first position in j[lo, hi) whose value is above c
__device__ __forceinline__ u64 ub32(const u32 *__restrict__ j, u64 lo, u64 hi, u32 c) {
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (j[mid] <= c) lo = mid + 1; else hi = mid; }
    return lo;
}
// the largest i in [lo, hi] with a[i] <= x (a[lo] <= x)
__device__ __forceinline__ u64 last_le(const u64 *__restrict__ a, u64 lo, u64 hi, u64 x) {
    while (lo < hi) { u64 mid = (lo + hi + 1) >> 1; if (a[mid] <= x) lo = mid; else hi = mid - 1; }
    return lo;
}

// The flop-balanced walk of a CTA over flops [lo, hi) (lo < hi) of the flat expansion behind cum, the scan of the lengths of
// entries [e_first, e_end): f(e, t) for every flop t, e the last of those entries with cum[e] <= t (t - cum[e] is the flop's
// place in entry e).  Thread 0 finds the CTA's first and last entry, then each warp takes 32 consecutive flops at a time and
// advances its lanes from one search.  Assumes 256-thread CTAs (8 warps); every thread of the CTA must call it.  f computes
// t - cum[e] itself: computed here, ahead of f's own loads, it changes the callers' code and register counts.
template <class F>
__device__ __forceinline__ void for_each_flop(const u64 *cum, u64 e_first, u64 e_end, u64 lo, u64 hi, F &&f) {
    __shared__ u64 s_e0, s_e1;
    const u32 tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        s_e0 = last_le(cum, e_first, e_end - 1, lo);
        s_e1 = last_le(cum, e_first, e_end - 1, hi - 1);
    }
    __syncthreads();
    const u64 e0 = s_e0, e1 = s_e1;
    for (u64 t0 = lo + (u64)warp * 32; t0 < hi; t0 += 8 * 32) {
        u64 e = last_le(cum, e0, e1, t0);
        const u64 t = t0 + lane;
        if (t < hi) {
            while (e < e1 && cum[e + 1] <= t) e++;
            f(e, t);
        }
    }
}
#endif

// ---- primitive wrappers implemented in prims.cu (CUB scan / sort) ----------------------------
void exclusive_scan_u64(const u64 *in, u64 *out, size_t n);           // out[i] = sum in[0..i)
void exclusive_scan_u32_to_u64(const u32 *in, u64 *out, size_t n);
void sort_keys_u64(u64 *keys_in_out, size_t n, int end_bit);            // ascending, in place (uses temp)
void sort_pairs_u64(u64 *keys_in_out, u64 *vals_in_out, size_t n, int end_bit); // stable
u64 reduce_sum_u64(const u64 *in, size_t n);
void sort_rows_u32(const u64 *rowptr, u64 nrows, u32 *cols, u64 nnz);  // every CSR row's entries ascending, in place (uses temp)

// ---- element-wise one-liners (prims.cu) ----
void iota_u64(u64 *p, u64 n);                     // p[i] = i
void fill_u64(u64 *p, u64 v, u64 n);
void fill_u32(u32 *p, u32 v, u64 n);
void widen_u32(const u32 *in, u64 *out, u64 n);
void narrow_u64(const u64 *in, u32 *out, u64 n);  // the low 32 bits

// ---- CSR results built from per-row counts (prims.cu) ----
// out emptied and shaped nrows x ncols, with room for its row pointers
void csr_shape(DevCSR &out, u64 nrows, u64 ncols);
// out's row pointers from the counts of its first `counted` rows (cnt holds out.nrows + 1 slots; the rest are zeroed here), then
// out.nnz and room for its column ids, and for its values when asked; returns out.nnz
u64 csr_rows_from_counts(u32 *cnt, u64 counted, DevCSR &out, bool values);

// ---- sorted u64 keys (prims.cu) ----
// head[e] = 1 where a run of equal keys of keys[0 .. n) starts (head[n] = 0), hpos its exclusive scan; returns the runs
u64 run_heads(const u64 *keys, u64 n, u32 *head, u64 *hpos);
// out[pos[i]] = in[i] for every i < n with flag[i]
void scatter_flagged(const u64 *in, u64 n, const u32 *flag, const u64 *pos, u64 *out);
// keys[0 .. n) sorted over end_bit bits and deduplicated (keys is replaced by the distinct keys); returns their count
u64 unique_sorted(DevBuf<u64> &keys, u64 n, int end_bit);
// the bits of x (0 for 0): a sort key holding every value <= x needs this end_bit
inline int bit_length(u64 x) { int b = 0; while (b < 64 && (x >> b)) b++; return b; }

} // namespace b200
