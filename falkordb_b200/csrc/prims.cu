// prims.cu -- context bring-up and the CUB-backed scan / radix-sort primitives.
// CUB (shipped with the CUDA toolkit) is used for the utility primitives only -- exclusive
// scans of row counts and the radix sort inside COO->CSR build / transpose; every kernel on the
// traversal hot path (mxm, frontier hops, materialise, eWise, BFS) is hand-written.
#include "common.cuh"
#include <cub/cub.cuh>
#include <thrust/iterator/transform_iterator.h>
#include <map>
#include <algorithm>
#include <mutex>
#include <thread>
#include <unordered_map>

namespace b200 {

Context &ctx() {
    static Context c;
    return c;
}

void ensure_init() {
    static std::mutex mu;
    Context &c = ctx();
    if (c.ready) return;
    std::lock_guard<std::mutex> lk(mu);
    if (c.ready) return;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        throw GrbError(-7002, "libb200grb: no CUDA device visible -- this backend has no CPU fallback");
    int dev = 0;
    CUDA_TRY(cudaGetDevice(&dev));
    c.device = dev;
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    c.num_sms = prop.multiProcessorCount;
    if (prop.l2CacheSize > 0) c.l2_bytes = (u64)prop.l2CacheSize;
    CUDA_TRY(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    c.ready = true;
}

// ---- small reads through mapped pinned memory (see common.cuh) -------------------------------------------------------
static const size_t SMALL_READ_MAX = 64, SMALL_SLOTS_BYTES = 8192;
static unsigned char *g_slots_host = nullptr, *g_slots_dev = nullptr;
static size_t g_slots_used = 0;
struct SmallPending { void *dst; size_t off, bytes; std::thread::id owner; };
static std::vector<SmallPending> g_small_pending;
static std::mutex g_small_mu;
__global__ void k_small_read(unsigned char *__restrict__ dst, const unsigned char *__restrict__ src, u32 bytes) {
    for (u32 i = threadIdx.x; i < bytes; i += 32) dst[i] = src[i];
}
bool small_read(void *dst, const void *src, size_t bytes) {
    if (bytes == 0 || bytes > SMALL_READ_MAX || !ctx().ready) return false;
    std::lock_guard<std::mutex> lk(g_small_mu);
    if (!g_slots_host) {
        if (cudaHostAlloc((void **)&g_slots_host, SMALL_SLOTS_BYTES, cudaHostAllocMapped) != cudaSuccess) { cudaGetLastError(); return false; }
        if (cudaHostGetDevicePointer((void **)&g_slots_dev, g_slots_host, 0) != cudaSuccess) { cudaGetLastError(); cudaFreeHost(g_slots_host); g_slots_host = nullptr; return false; }
    }
    size_t off = (g_slots_used + 15) & ~(size_t)15;
    if (off + bytes > SMALL_SLOTS_BYTES) return false;
    g_slots_used = off + bytes;
    k_small_read<<<1, 32, 0, stream()>>>(g_slots_dev + off, (const unsigned char *)src, (u32)bytes);
    if (cudaGetLastError() != cudaSuccess) { g_slots_used = off; return false; }
    g_small_pending.push_back({dst, off, bytes, std::this_thread::get_id()});
    return true;
}
void drop_small_reads() {
    std::lock_guard<std::mutex> lk(g_small_mu);
    // only the caller's own reads: another thread's destinations are alive.  Slots stay reserved until the next flush resets
    // the bump pointer (the kernels may still be in flight).
    const std::thread::id me = std::this_thread::get_id();
    g_small_pending.erase(std::remove_if(g_small_pending.begin(), g_small_pending.end(),
                                         [&](const SmallPending &p) { return p.owner == me; }), g_small_pending.end());
}
void flush_small_reads() {
    std::lock_guard<std::mutex> lk(g_small_mu);
    for (const SmallPending &p : g_small_pending) memcpy(p.dst, g_slots_host + p.off, p.bytes);
    g_small_pending.clear();
    g_slots_used = 0;
}

// ---- caching allocator ----------------------------------------------------------------------------------
static std::mutex g_pool_mu;
static std::map<size_t, std::vector<void *>> g_free;     // class size -> cached blocks
static std::unordered_map<void *, size_t> g_size;        // live + cached block -> class size
static size_t g_cached_bytes = 0;

static size_t size_class(size_t b) {
    if (b <= 512) return 512;
    size_t p = 1;
    while (p < b) p <<= 1;                 // next power of two
    if (b <= ((size_t)1 << 20)) return p;
    size_t step = p >> 4;                  // above 1 MiB: 1/16-of-a-power-of-two granularity (<= 6.7% slack)
    return (b + step - 1) / step * step;
}
void pool_trim() {
    std::lock_guard<std::mutex> lk(g_pool_mu);
    cudaStreamSynchronize(stream());
    for (auto &kv : g_free) for (void *p : kv.second) { cudaFree(p); g_size.erase(p); }
    g_free.clear();
    g_cached_bytes = 0;
}
size_t pool_bytes_cached() { return g_cached_bytes; }
void *pool_alloc(size_t bytes) {
    size_t cls = size_class(bytes);
    {
        std::lock_guard<std::mutex> lk(g_pool_mu);
        // exact class first; large requests also take the smallest cached block of up to twice the size, so a result
        // buffer whose size drifts from step to step (nnz of a frontier batch) reuses one block instead of growing a new
        // multi-GB cudaMalloc per size class (each costs milliseconds inside a timed step)
        const size_t limit = cls >= ((size_t)1 << 20) ? cls * 2 : cls;
        for (auto it = g_free.lower_bound(cls); it != g_free.end() && it->first <= limit; ++it) {
            if (it->second.empty()) continue;
            void *p = it->second.back();
            it->second.pop_back();
            g_cached_bytes -= it->first;
            return p;
        }
    }
    void *p = nullptr;
    const size_t want = cls;
    if (cls >= ((size_t)256 << 20)) cls = size_class(cls + cls / 4);   // headroom: the next, slightly larger, request fits too
    cudaError_t e = cudaMalloc(&p, cls);
    if (e == cudaErrorMemoryAllocation) {  // give cached blocks back to the driver and retry once, without the headroom
        cudaGetLastError();
        pool_trim();
        cls = want;
        e = cudaMalloc(&p, cls);
    }
    if (e != cudaSuccess) throw CudaError(e, __FILE__, __LINE__);
    std::lock_guard<std::mutex> lk(g_pool_mu);
    g_size[p] = cls;
    return p;
}
void pool_free(void *p) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(g_pool_mu);
    auto it = g_size.find(p);
    if (it == g_size.end()) { cudaFree(p); return; }
    g_free[it->second].push_back(p);
    g_cached_bytes += it->second;
}

// ---- per-kernel timing registry ------------------------------------------------------------------
struct TimedRec { int id; cudaEvent_t e0, e1; u64 bytes; };
static std::vector<TimedRec> g_recs;
static std::vector<cudaEvent_t> g_event_pool;
static std::mutex g_timed_mu;
static cudaEvent_t g_open[TK_COUNT_];
static double g_ms[TK_COUNT_];
static u64 g_n[TK_COUNT_], g_bytes[TK_COUNT_];

const char *timed_name(int id) {
    static const char *names[] = {"bits_pull", "bits_push", "heavy_accumulate", "small_rows", "bits_fill",
                                  "bits_count", "bitmap_expand", "bfs_expand", "union", "filter", "mxv_fp64", "spgemm_masked", "transpose",
                                  "bits_delta", "bits_repair", "bits_pull_acc", "bits_push_acc", "edge_expand", "bfs_delta", "adj_build",
                                  "tensor_write", "var_len_trails", "var_len_reach_both", "shortest_path",
                                  "all_shortest_paths"};
    return (id >= 0 && id < TK_COUNT_) ? names[id] : "?";
}
static cudaEvent_t get_event() {
    if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
    cudaEvent_t e;
    CUDA_TRY(cudaEventCreate(&e));
    return e;
}
void timed_begin(int id) {
    if (!ctx().opt_timing) return;
    std::lock_guard<std::mutex> lk(g_timed_mu);
    cudaEvent_t e = get_event();
    CUDA_TRY(cudaEventRecord(e, stream()));
    g_open[id] = e;
}
void timed_end(int id, u64 bytes) noexcept {
    // runs from ~TimedScope, possibly while a CUDA error is unwinding: it must never throw.  A failed record drops the sample.
    if (!ctx().opt_timing) return;
    try {
        std::lock_guard<std::mutex> lk(g_timed_mu);
        if (!g_open[id]) return;
        cudaEvent_t e0 = g_open[id];
        g_open[id] = nullptr;
        cudaEvent_t e = get_event();
        if (cudaEventRecord(e, stream()) != cudaSuccess) {
            cudaGetLastError();
            g_event_pool.push_back(e0);
            g_event_pool.push_back(e);
            return;
        }
        g_recs.push_back(TimedRec{id, e0, e, bytes});
    } catch (...) {
    }
}
static void drain_locked() {
    if (g_recs.empty()) return;
    CUDA_TRY(cudaStreamSynchronize(stream()));
    for (TimedRec &r : g_recs) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) { g_ms[r.id] += ms; g_n[r.id]++; g_bytes[r.id] += r.bytes; }
        g_event_pool.push_back(r.e0);
        g_event_pool.push_back(r.e1);
    }
    g_recs.clear();
}
void timed_collect(double *ms, u64 *launches, u64 *bytes) {
    std::lock_guard<std::mutex> lk(g_timed_mu);
    drain_locked();
    for (int i = 0; i < TK_COUNT_; i++) { ms[i] = g_ms[i]; launches[i] = g_n[i]; bytes[i] = g_bytes[i]; }
}
void timed_reset() {
    std::lock_guard<std::mutex> lk(g_timed_mu);
    drain_locked();
    for (int i = 0; i < TK_COUNT_; i++) { g_ms[i] = 0; g_n[i] = 0; g_bytes[i] = 0; }
}

void exclusive_scan_u64(const u64 *in, u64 *out, size_t n) {
    if (n == 0) return;
    size_t tb = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, n, stream()));
    DevBuf<char> tmp(tb);
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.ptr, tb, in, out, n, stream()));
    ctx().lib_launches += 2;
}

struct U32ToU64 {
    __host__ __device__ u64 operator()(u32 v) const { return (u64)v; }
};

void exclusive_scan_u32_to_u64(const u32 *in, u64 *out, size_t n) {
    if (n == 0) return;
    auto it = thrust::make_transform_iterator(in, U32ToU64());
    size_t tb = 0;
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, it, out, n, stream()));
    DevBuf<char> tmp(tb);
    CUDA_TRY(cub::DeviceScan::ExclusiveSum(tmp.ptr, tb, it, out, n, stream()));
    ctx().lib_launches += 2;
}

void sort_keys_u64(u64 *keys, size_t n, int end_bit) {
    if (n <= 1) return;
    DevBuf<u64> alt(n);
    cub::DoubleBuffer<u64> db(keys, alt.ptr);
    if ((u64)n > 0x7fffffffULL) throw GrbError(-8, "sort_keys_u64: more than 2^31-1 keys not supported yet");
    size_t tb = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortKeys(nullptr, tb, db, (int)n, 0, end_bit, stream()));
    DevBuf<char> tmp(tb);
    CUDA_TRY(cub::DeviceRadixSort::SortKeys(tmp.ptr, tb, db, (int)n, 0, end_bit, stream()));
    if (db.Current() != keys) d2d(keys, db.Current(), n);
    ctx().lib_launches += 8;
}

void sort_pairs_u64(u64 *keys, u64 *vals, size_t n, int end_bit) {
    if (n <= 1) return;
    if ((u64)n > 0x7fffffffULL) throw GrbError(-8, "sort_pairs_u64: more than 2^31-1 keys not supported yet");
    DevBuf<u64> altk(n), altv(n);
    cub::DoubleBuffer<u64> dk(keys, altk.ptr), dv(vals, altv.ptr);
    size_t tb = 0;
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, dk, dv, (int)n, 0, end_bit, stream()));
    DevBuf<char> tmp(tb);
    CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.ptr, tb, dk, dv, (int)n, 0, end_bit, stream()));
    if (dk.Current() != keys) d2d(keys, dk.Current(), n);
    if (dv.Current() != vals) d2d(vals, dv.Current(), n);
    ctx().lib_launches += 8;
}

// Sorts the entries of every CSR row: one radix sort of (row, entry) keys over the row-index bits and the entry's 32.  Rows
// keep their extents, so the sorted low words go straight back.  16 * nnz bytes of temporaries, released on return.
__global__ void k_row_keys(const u64 *__restrict__ rowptr, u64 nrows, const u32 *__restrict__ cols, u64 *__restrict__ keys) {
    const u64 nwarps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u32 lane = threadIdx.x & 31;
    for (u64 r = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < nrows; r += nwarps)
        for (u64 q = rowptr[r] + lane; q < rowptr[r + 1]; q += 32) keys[q] = (r << 32) | cols[q];
}
void sort_rows_u32(const u64 *rowptr, u64 nrows, u32 *cols, u64 nnz) {
    if (nnz <= 1) return;
    if (nrows > ((u64)1 << 32)) throw GrbError(-8, "sort_rows_u32: more than 2^32 rows not supported");
    DevBuf<u64> keys(nnz);
    LAUNCH(k_row_keys, grid_for(nrows * 32, 256, (u64)ctx().num_sms * 32), 256, 0, rowptr, nrows, cols, keys.ptr);
    int row_bits = 1;
    while (row_bits < 32 && ((u64)1 << row_bits) < nrows) row_bits++;
    sort_keys_u64(keys.ptr, nnz, 32 + row_bits);
    narrow_u64(keys.ptr, cols, nnz);
}

__global__ void k_iota_u64(u64 *__restrict__ v, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) v[i] = i;
}
template <class T>
__global__ void k_fill(T *__restrict__ p, T v, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void k_widen_u32(const u32 *__restrict__ in, u64 *__restrict__ out, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) out[i] = in[i];
}
__global__ void k_narrow_u64(const u64 *__restrict__ in, u32 *__restrict__ out, u64 n) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) out[i] = (u32)in[i];
}
static u32 small_grid(u64 n) { return grid_for(n, 256, (u64)ctx().num_sms * 16); }
void iota_u64(u64 *p, u64 n) { if (n) LAUNCH(k_iota_u64, small_grid(n), 256, 0, p, n); }
void fill_u64(u64 *p, u64 v, u64 n) { if (n) LAUNCH(k_fill<u64>, small_grid(n), 256, 0, p, v, n); }
void fill_u32(u32 *p, u32 v, u64 n) { if (n) LAUNCH(k_fill<u32>, small_grid(n), 256, 0, p, v, n); }
void widen_u32(const u32 *in, u64 *out, u64 n) { if (n) LAUNCH(k_widen_u32, small_grid(n), 256, 0, in, out, n); }
void narrow_u64(const u64 *in, u32 *out, u64 n) { if (n) LAUNCH(k_narrow_u64, small_grid(n), 256, 0, in, out, n); }

void csr_shape(DevCSR &out, u64 nrows, u64 ncols) {
    out.clear();
    out.nrows = nrows; out.ncols = ncols;
    out.p.alloc(nrows + 1);
}
u64 csr_rows_from_counts(u32 *cnt, u64 counted, DevCSR &out, bool values) {
    CUDA_TRY(cudaMemsetAsync(cnt + counted, 0, (out.nrows + 1 - counted) * sizeof(u32), stream()));
    exclusive_scan_u32_to_u64(cnt, out.p.ptr, out.nrows + 1);
    out.nnz = read_scalar(out.p.ptr + out.nrows);
    out.j.alloc(out.nnz);
    if (values) out.x.alloc(out.nnz);
    return out.nnz;
}

__global__ void k_run_heads(const u64 *__restrict__ k, u64 n, u32 *__restrict__ head) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e <= n; e += (u64)gridDim.x * blockDim.x)
        head[e] = e < n && (e == 0 || k[e] != k[e - 1]) ? 1 : 0;
}
__global__ void k_scatter_flagged(const u64 *__restrict__ in, u64 n, const u32 *__restrict__ flag, const u64 *__restrict__ pos,
                                  u64 *__restrict__ out) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        if (flag[i]) out[pos[i]] = in[i];
}
u64 run_heads(const u64 *keys, u64 n, u32 *head, u64 *hpos) {
    LAUNCH(k_run_heads, grid_for(n + 1, 256), 256, 0, keys, n, head);
    exclusive_scan_u32_to_u64(head, hpos, n + 1);
    return read_scalar(hpos + n);
}
void scatter_flagged(const u64 *in, u64 n, const u32 *flag, const u64 *pos, u64 *out) {
    LAUNCH(k_scatter_flagged, grid_for(n, 256), 256, 0, in, n, flag, pos, out);
}
u64 unique_sorted(DevBuf<u64> &keys, u64 n, int end_bit) {
    if (!n) return 0;
    sort_keys_u64(keys.ptr, n, end_bit);
    DevBuf<u32> head(n + 1);
    DevBuf<u64> hpos(n + 1), out;
    const u64 m = run_heads(keys.ptr, n, head.ptr, hpos.ptr);
    out.alloc(m);
    scatter_flagged(keys.ptr, n, head.ptr, hpos.ptr, out.ptr);
    keys = std::move(out);
    return m;
}

u64 reduce_sum_u64(const u64 *in, size_t n) {
    if (n == 0) return 0;
    DevBuf<u64> out(1);
    size_t tb = 0;
    CUDA_TRY(cub::DeviceReduce::Sum(nullptr, tb, in, out.ptr, n, stream()));
    DevBuf<char> tmp(tb);
    CUDA_TRY(cub::DeviceReduce::Sum(tmp.ptr, tb, in, out.ptr, n, stream()));
    ctx().lib_launches += 2;
    return read_scalar(out.ptr);
}

} // namespace b200
