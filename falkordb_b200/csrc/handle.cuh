// handle.cuh -- what the C ABI (grb_api.cu) and the batched relationship calls (graph_api.cu) share: the matrix handle and the
// host allocator behind it, error reporting, locking, and the form-management and dispatch helpers grb_api.cu defines.
#pragma once
#include "../../include/b200grb.h"
#include "common.cuh"
#include "ops.cuh"
#include <algorithm>
#include <atomic>
#include <mutex>
#include <string>
#include <vector>

using namespace b200;

enum { T_BOOL = 1, T_UINT64 = 2, T_INT64 = 3, T_UINT32 = 4, T_FP64 = 5 };   // FP64 values travel as IEEE-754 bit patterns in the u64 arrays

// the allocator given to GxB_init and the host footprint allocated through it (grb_api.cu).  The globals shared by the two sources
// are hidden: the library exports C ABI names only.
extern __attribute__((visibility("hidden"))) void *(*g_user_malloc)(size_t);
extern __attribute__((visibility("hidden"))) void (*g_user_free)(void *);
extern __attribute__((visibility("hidden"))) std::atomic<uint64_t> g_host_bytes, g_host_allocs;
template <class T> struct UAlloc {
    typedef T value_type;
    UAlloc() noexcept {}
    template <class U> UAlloc(const UAlloc<U> &) noexcept {}
    T *allocate(size_t n) {
        if (n > (size_t)-1 / sizeof(T)) throw std::bad_alloc();
        const size_t bytes = n * sizeof(T);
        void *p = g_user_malloc(bytes > 0 ? bytes : 1);
        if (!p) throw std::bad_alloc();
        g_host_bytes += n * sizeof(T); g_host_allocs++;
        return (T *)p;
    }
    void deallocate(T *p, size_t n) noexcept { g_host_bytes -= n * sizeof(T); g_user_free(p); }
    template <class U> bool operator==(const UAlloc<U> &) const noexcept { return true; }
    template <class U> bool operator!=(const UAlloc<U> &) const noexcept { return false; }
};
template <class T> using uvec = std::vector<T, UAlloc<T>>;
// handles: operator new / delete through the same hooks
struct UObject {
    static void *operator new(size_t n) {
        void *p = g_user_malloc(n);
        if (!p) throw std::bad_alloc();
        g_host_bytes += n; g_host_allocs++;
        return p;
    }
    static void operator delete(void *p, size_t n) noexcept { if (p) { g_host_bytes -= n; g_user_free(p); } }
};

struct HostStore {
    uvec<u64> hrow; // ascending ids of the non-empty rows
    uvec<u64> hptr; // hrow.size()+1
    uvec<u64> hcol; // ascending inside a row
    uvec<u64> hval; // empty for pattern-only (BOOL)
    void clear() { hrow.clear(); hptr.assign(1, 0); hcol.clear(); hval.clear(); }
    u64 nnz() const { return hcol.size(); }
};
struct PendingOp { u64 i, j, v; u64 seq; bool del; };

static const u32 MAGIC = 0xB200A7u;

struct GB_Matrix_opaque : UObject {
    u32 magic = MAGIC;
    int type = T_BOOL;
    u64 nrows = 0, ncols = 0;
    std::mutex mu;
    bool host_valid = true;
    HostStore host;
    uvec<PendingOp> pending;
    bool dev_valid = false;
    DevCSR dev;
    bool bits_valid = false;
    u64 bits_nv = ~0ULL;   // nvals of `bits` once counted (~0 = not yet)
    int diag_state = -1;   // -1 unknown, 0 no, 1 the device CSR is a diagonal matrix (label matrix): mxm by it is a column filter
    DevBits bits;
    bool devT_valid = false;
    DevCSR devT;
    PullTables pt;   // pull-direction tables of devT (bits_hop.cu)
    DevBuf<u32> bfs_deg; u64 bfs_edges = 0; bool bfs_deg_valid = false;   // out-degree table of the BFS engine (bfs_do.cu)
    DevIdStore ids;  // device copy of the host store, for a Tensor's multi-edge layers (B200_expand_edges)
    int sparsity_control = GxB_HYPERSPARSE | GxB_SPARSE | GxB_BITMAP | GxB_FULL;
    int hyper_hash = 1;
    int orientation = GrB_ROWMAJOR;
    GB_Matrix_opaque() { host.clear(); }
    bool valued() const { return type != T_BOOL; }
};

// ------------------------------------------------------------------------------------------------ errors
extern __attribute__((visibility("hidden"))) thread_local std::string tl_error;
extern __attribute__((visibility("hidden"))) std::mutex g_gpu_mu;
// Holds g_gpu_mu for one bulk operation.  If the operation unwinds with an exception, small reads whose destinations lived on
// the abandoned stack are forgotten BEFORE the mutex is released: once another thread owns the mutex its sync_stream() would
// otherwise deliver into dead frames.
struct GpuLock {
    std::unique_lock<std::mutex> lk;
    int entry;
    GpuLock() : lk(g_gpu_mu), entry(std::uncaught_exceptions()) {}
    ~GpuLock() { if (std::uncaught_exceptions() > entry) drop_small_reads(); }
};

template <class F>
static GrB_Info guarded(F &&f) {
    // an exception may unwind past a small read whose destination lived on the abandoned stack: forget such reads
    // (drop_small_reads) so that the next sync_stream() does not deliver into dead frames
    try {
        return f();
    } catch (const GrbError &e) {
        drop_small_reads();
        tl_error = e.what();
        return (GrB_Info)e.info;
    } catch (const CudaError &e) {
        drop_small_reads();
        tl_error = e.what();
        if (e.code == cudaErrorMemoryAllocation) return GrB_OUT_OF_MEMORY;
        return GxB_GPU_ERROR;
    } catch (const std::bad_alloc &) {
        drop_small_reads();
        tl_error = "host allocation failed";
        return GrB_OUT_OF_MEMORY;
    } catch (const std::exception &e) {
        drop_small_reads();
        tl_error = e.what();
        return GrB_PANIC;
    }
}
#define CHECK_PTR(p) do { if (!(p)) { tl_error = "null pointer: " #p; return GrB_NULL_POINTER; } } while (0)
#define CHECK_MAT(m) do { if (!(m)) { tl_error = "null matrix: " #m; return GrB_NULL_POINTER; } \
                          if ((m)->magic != MAGIC) { tl_error = "invalid matrix: " #m; return GrB_INVALID_OBJECT; } } while (0)

struct MultiLock {
    uvec<std::unique_lock<std::mutex>> locks;
    MultiLock(std::initializer_list<GrB_Matrix> ms) : MultiLock(ms.begin(), ms.end()) {}
    template <class It> MultiLock(It first, It last) {
        uvec<GrB_Matrix> v;
        for (; first != last; ++first) if (*first) v.push_back(*first);
        std::sort(v.begin(), v.end());
        v.erase(std::unique(v.begin(), v.end()), v.end());
        for (GrB_Matrix m : v) locks.emplace_back(m->mu);
    }
};

struct Desc { bool t0 = false, t1 = false, comp = false, structure = false, replace = false; };

// ------------------------------------------------------------------------------------------------ form management and dispatch
// Defined in grb_api.cu.  frontier_product, frontier_mxm and bfs_staged sit inside its extern "C" block, hence extern "C++"
// at their definitions.
void set_dev(GrB_Matrix A, DevCSR &&d);
void set_bits(GrB_Matrix A, DevBits &&b);
void finish_pending(GrB_Matrix A);
void ensure_dev(GrB_Matrix A);
void ensure_devT(GrB_Matrix A);
void ensure_bits(GrB_Matrix A);
void ensure_host(GrB_Matrix A);
u64 matrix_nvals(GrB_Matrix A);
bool is_huge(GrB_Matrix A);
bool frontier_product(GrB_Matrix A, GrB_Matrix B, bool pt_ok, DevBits &Y, u64 *fl, int *path, bool acc = false);
bool frontier_mxm(GrB_Matrix C, GrB_Matrix Mask, GrB_Matrix A, GrB_Matrix B, const Desc &d, bool accum,
                  const DevCSR *dm = nullptr, const DevCSR *dp = nullptr);
void bfs_staged(GrB_Matrix A, const DevCSR *AT, u64 n, u64 lo, BfsComm *comm, u64 src, i64 max_level, i64 dest,
                i64 *level, i64 *parent, int location, B200_BfsInfo *info_out,
                const std::vector<BfsOperand> *dirty = nullptr, const u32 *deg = nullptr, u64 total_edges = 0);
