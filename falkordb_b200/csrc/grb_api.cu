// grb_api.cu -- the C ABI (include/b200grb.h): opaque handles, GraphBLAS write-back semantics
// (mask / complement / structural / replace / accum) and dispatch onto the CUDA kernel layer.
//
// Handle model.  A GrB_Matrix owns up to three interchangeable forms of the same content:
//   host  : hypersparse sorted tuples (element access, iterators, pending setElement/removeElement)
//   dev   : device CSR (every bulk operation)
//   bits  : device frontier bit-matrix (short-fat mxm results between hops, bits.cu)
// plus a cached transpose mirror of `dev` for the pull direction.  Bulk results are produced on the
// device and only travel to the host when something observes them (GraphBLAS non-blocking mode:
// matrix.rs:116-131 initialises GrB_NONBLOCKING).  There is NO CPU implementation of any bulk
// operation in this file: without a GPU they fail with GxB_GPU_ERROR.
#include "handle.cuh"
#include <cstring>
#include <memory>

// ------------------------------------------------------------------------------------------------ opaque types
struct GB_Type_opaque { int code; size_t size; const char *name; };
struct GB_UnaryOp_opaque { int code; };
struct GB_BinaryOp_opaque { int code; };
struct GB_Semiring_opaque { int code; };
struct GB_Global_opaque { int x; };
struct GB_Descriptor_opaque { bool t0, t1, comp, structure, replace; };
struct GB_Scalar_opaque { int type; bool has; uint64_t val; };   // allocated with the C++ allocator: 24 bytes, short-lived

enum { OP_ANY_BOOL = 1, OP_SECOND_UINT64 = 2, OP_ANY_UINT64 = 3, OP_PLUS_FP64 = 4 };
enum { SR_ANY_PAIR = 1, SR_PLUS_TIMES_FP64 = 2, SR_PLUS_SECOND_FP64 = 3 };

static GB_Type_opaque t_bool = {T_BOOL, 1, "bool"}, t_u64 = {T_UINT64, 8, "uint64_t"}, t_i64 = {T_INT64, 8, "int64_t"},
                      t_u32 = {T_UINT32, 4, "uint32_t"}, t_f64 = {T_FP64, 8, "double"};
static GB_Semiring_opaque s_any_pair = {SR_ANY_PAIR}, s_plus_times_f64 = {SR_PLUS_TIMES_FP64}, s_plus_second_f64 = {SR_PLUS_SECOND_FP64};
static GB_BinaryOp_opaque b_any_bool = {OP_ANY_BOOL}, b_second_u64 = {OP_SECOND_UINT64}, b_any_u64 = {OP_ANY_UINT64}, b_plus_f64 = {OP_PLUS_FP64};
static GB_UnaryOp_opaque u_one_bool = {1};
static GB_Global_opaque g_global = {0};

extern "C" {
GrB_Type GrB_BOOL = &t_bool, GrB_UINT64 = &t_u64, GrB_INT64 = &t_i64, GrB_UINT32 = &t_u32, GrB_FP64 = &t_f64;
GrB_Semiring GxB_ANY_PAIR_BOOL = &s_any_pair, GrB_PLUS_TIMES_SEMIRING_FP64 = &s_plus_times_f64, GxB_PLUS_SECOND_FP64 = &s_plus_second_f64;
GrB_BinaryOp GxB_ANY_BOOL = &b_any_bool, GrB_SECOND_UINT64 = &b_second_u64, GxB_ANY_UINT64 = &b_any_u64, GrB_PLUS_FP64 = &b_plus_f64;
GrB_UnaryOp GxB_ONE_BOOL = &u_one_bool;
const GrB_Global GrB_GLOBAL = &g_global;
}

#define DESC(name, R, S, C, T0, T1) \
    static GB_Descriptor_opaque d_##name = {T0, T1, C, S, R}; \
    extern "C" { GrB_Descriptor GrB_DESC_##name = &d_##name; }
DESC(T1, 0, 0, 0, 0, 1) DESC(T0, 0, 0, 0, 1, 0) DESC(T0T1, 0, 0, 0, 1, 1)
DESC(C, 0, 0, 1, 0, 0) DESC(CT1, 0, 0, 1, 0, 1) DESC(CT0, 0, 0, 1, 1, 0) DESC(CT0T1, 0, 0, 1, 1, 1)
DESC(S, 0, 1, 0, 0, 0) DESC(ST1, 0, 1, 0, 0, 1) DESC(ST0, 0, 1, 0, 1, 0) DESC(ST0T1, 0, 1, 0, 1, 1)
DESC(SC, 0, 1, 1, 0, 0) DESC(SCT1, 0, 1, 1, 0, 1) DESC(SCT0, 0, 1, 1, 1, 0) DESC(SCT0T1, 0, 1, 1, 1, 1)
DESC(R, 1, 0, 0, 0, 0) DESC(RT1, 1, 0, 0, 0, 1) DESC(RT0, 1, 0, 0, 1, 0) DESC(RT0T1, 1, 0, 0, 1, 1)
DESC(RC, 1, 0, 1, 0, 0) DESC(RCT1, 1, 0, 1, 0, 1) DESC(RCT0, 1, 0, 1, 1, 0) DESC(RCT0T1, 1, 0, 1, 1, 1)
DESC(RS, 1, 1, 0, 0, 0) DESC(RST1, 1, 1, 0, 0, 1) DESC(RST0, 1, 1, 0, 1, 0) DESC(RST0T1, 1, 1, 0, 1, 1)
DESC(RSC, 1, 1, 1, 0, 0) DESC(RSCT1, 1, 1, 1, 0, 1) DESC(RSCT0, 1, 1, 1, 1, 0) DESC(RSCT0T1, 1, 1, 1, 1, 1)

// ---- host memory goes through the allocator given to GxB_init (matrix.rs:123-131: Redis' allocator, so that the server's
// memory accounting and QUERY_MEM_CAPACITY see this library's host footprint).  Every host container of a handle (tuple
// stores, pending lists, vector payloads, iterator snapshots) and the handles themselves use it; so do the buffers handed
// to the caller (unloaded arrays, blobs), which the caller frees with the same allocator (vector.rs:171-172).
void *(*g_user_malloc)(size_t) = malloc;
static void *(*g_user_calloc)(size_t, size_t) = calloc;
static void *(*g_user_realloc)(void *, size_t) = realloc;
void (*g_user_free)(void *) = free;
std::atomic<uint64_t> g_host_bytes{0}, g_host_allocs{0};     // live bytes / allocation calls through the hooks
static void *user_zalloc(size_t bytes) {        // zero-initialised block (the container struct); calloc hook when the caller gave one
    void *p = g_user_calloc ? g_user_calloc(1, bytes) : g_user_malloc(bytes);
    if (p && !g_user_calloc) memset(p, 0, bytes);
    return p;
}
static void *user_grow(void *old, size_t old_bytes, size_t new_bytes) {   // realloc hook when given, else malloc + copy + free
    if (g_user_realloc) return g_user_realloc(old, new_bytes);
    void *p = g_user_malloc(new_bytes);
    if (p && old) { memcpy(p, old, old_bytes < new_bytes ? old_bytes : new_bytes); g_user_free(old); }
    return p;
}
// the hooks as the host-side mirror and the tests see them
extern "C" void *B200_user_realloc(void *p, size_t old_bytes, size_t new_bytes) { return user_grow(p, old_bytes, new_bytes); }

struct GB_Vector_opaque : UObject {
    u32 magic = MAGIC;
    int type = T_BOOL;
    u64 n = 0;
    uvec<u64> idx; // ascending
    uvec<i64> val; // same length (bool: 1)
    // full (dense) form of the GxB_Container payload vectors: n entries of `type` in fx (user allocator), idx / val unused
    bool full = false;
    void *fx = nullptr;
    u64 fbytes = 0;
};

struct GB_Iterator_opaque : UObject {
    GrB_Vector V = nullptr;   // vector mode (GxB_Vector_Iterator_*): k = position of the current entry, pmax = nvals
    GrB_Matrix A = nullptr;
    u64 k = 0; // vector (non-empty row) position; the row itself in bitmap mode
    u64 q = 0; // entry position; the column itself in bitmap mode
    bool exhausted = true;
    // bitmap mode: a dense frontier-chain result is walked from a row-major packed bitmap snapshot (1 bit per slot over
    // PCIe instead of a 64-bit column index per entry); same ascending (row, col) order as the sparse walk
    bool bitmap = false;
    u64 wpr = 0, nrows = 0, ncols = 0;
    uvec<u64> bm;
    // first set bit of `row` at column >= from, or ncols
    u64 first_set(u64 row, u64 from) const {
        if (from >= ncols) return ncols;
        const u64 *w = bm.data() + row * wpr;
        u64 i = from >> 6;
        u64 cur = w[i] & (~0ULL << (from & 63));
        while (true) {
            if (cur) { u64 c = (i << 6) + (u64)__builtin_ctzll(cur); return c < ncols ? c : ncols; }
            if (++i >= wpr) return ncols;
            cur = w[i];
        }
    }
};

// ------------------------------------------------------------------------------------------------ errors
thread_local std::string tl_error;
std::mutex g_gpu_mu; // serialises GPU submission across caller threads

// ------------------------------------------------------------------------------------------------ form management
static void invalidate_aux(GrB_Matrix A) {
    A->diag_state = -1;
    A->bfs_deg.release(); A->bfs_deg_valid = false; A->bfs_edges = 0;
    A->devT_valid = false;
    A->devT.clear();
    A->pt.clear();
    // every change of the stored entries passes through here: set_dev / set_bits / set_empty (clear, build, element-wise
    // results, container load / unload), finish_pending (setElement / removeElement) and resize
    A->ids.clear();
}

void set_dev(GrB_Matrix A, DevCSR &&d) {
    A->dev = std::move(d);
    A->dev.nrows = A->nrows; A->dev.ncols = A->ncols;
    // type discipline: BOOL is pattern-only, UINT64/INT64 always carry a value array
    if (!A->valued()) A->dev.x.release();
    else if (!A->dev.has_values()) {
        A->dev.x.alloc(A->dev.nnz);
        fill_u64(A->dev.x.ptr, A->type == T_FP64 ? 0x3FF0000000000000ULL : 1ULL, A->dev.nnz); // typecast of `true` (1 / 1.0)
    }
    A->dev_valid = true;
    A->host_valid = false;
    A->host.clear();
    A->pending.clear();
    A->bits_valid = false;
    A->bits.clear();
    invalidate_aux(A);
}

void set_bits(GrB_Matrix A, DevBits &&b) {
    A->bits = std::move(b);
    A->bits_nv = ~0ULL;
    A->bits_valid = true;
    A->dev_valid = false;
    A->dev.clear();
    A->host_valid = false;
    A->host.clear();
    A->pending.clear();
    invalidate_aux(A);
}

// a frontier kept in another matrix's hot-set order (bits_hop.cu: permuted form) goes back to natural vertex order before anything
// but the pull it was ordered for looks at it
static void natural_bits(GrB_Matrix A) {
    if (A->bits_valid && A->bits.permuted()) bits_naturalise(A->bits);
}

static void set_empty(GrB_Matrix A) {
    A->host.clear();
    A->host_valid = true;
    A->pending.clear();
    A->dev_valid = false; A->dev.clear();
    A->bits_valid = false; A->bits.clear();
    invalidate_aux(A);
}

static void download_to_host(GrB_Matrix A); // fwd

// apply queued setElement / removeElement onto the host store (GrB_Matrix_wait, matrix.rs:781-796)
void finish_pending(GrB_Matrix A) {
    if (A->pending.empty()) return;
    if (!A->host_valid) download_to_host(A);
    uvec<PendingOp> &p = A->pending;
    std::sort(p.begin(), p.end(), [](const PendingOp &a, const PendingOp &b) {
        if (a.i != b.i) return a.i < b.i;
        if (a.j != b.j) return a.j < b.j;
        return a.seq < b.seq;
    });
    // keep the last op per coordinate
    uvec<PendingOp> last;
    last.reserve(p.size());
    for (size_t t = 0; t < p.size(); t++)
        if (t + 1 == p.size() || p[t + 1].i != p[t].i || p[t + 1].j != p[t].j) last.push_back(p[t]);
    HostStore &h = A->host;
    HostStore out;
    out.hptr.clear();
    bool valued = A->valued();
    size_t pi = 0;
    u64 k = 0, nvec = h.hrow.size();
    auto emit = [&](u64 row, u64 col, u64 val) {
        if (out.hrow.empty() || out.hrow.back() != row) { out.hrow.push_back(row); out.hptr.push_back(out.hcol.size()); }
        out.hcol.push_back(col);
        if (valued) out.hval.push_back(val);
    };
    while (k < nvec || pi < last.size()) {
        u64 row;
        if (k >= nvec) row = last[pi].i;
        else if (pi >= last.size()) row = h.hrow[k];
        else row = std::min(h.hrow[k], last[pi].i);
        u64 q = 0, qe = 0;
        if (k < nvec && h.hrow[k] == row) { q = h.hptr[k]; qe = h.hptr[k + 1]; k++; }
        while (q < qe || (pi < last.size() && last[pi].i == row)) {
            bool hp = pi < last.size() && last[pi].i == row;
            if (q < qe && (!hp || h.hcol[q] < last[pi].j)) {
                emit(row, h.hcol[q], valued ? h.hval[q] : 1);
                q++;
            } else {
                const PendingOp &op = last[pi];
                if (q < qe && h.hcol[q] == op.j) q++; // overwritten or deleted
                if (!op.del) emit(row, op.j, op.v);
                pi++;
            }
        }
    }
    out.hptr.push_back(out.hcol.size());
    A->host = std::move(out);
    A->pending.clear();
    A->dev_valid = false; A->dev.clear();
    A->bits_valid = false; A->bits.clear();
    invalidate_aux(A);
}

static void upload_to_dev(GrB_Matrix A) {
    if (A->nrows >= ((u64)1 << 32) || A->ncols >= ((u64)1 << 32))
        throw GrbError(GrB_NOT_IMPLEMENTED, "bulk GPU operations need dimensions < 2^32 (host-only hypersparse matrix)");
    ensure_init();
    HostStore &h = A->host;
    u64 nvec = h.hrow.size(), nnz = h.nnz();
    DevCSR d;
    d.nrows = A->nrows; d.ncols = A->ncols; d.nnz = nnz;
    d.p.alloc(A->nrows + 1);
    if (nnz == 0) {
        d.p.zero();
    } else {
        DevBuf<u64> dh(nvec), dp(nvec + 1), dc(nnz);
        h2d(dh.ptr, h.hrow.data(), nvec);
        h2d(dp.ptr, h.hptr.data(), nvec + 1);
        h2d(dc.ptr, h.hcol.data(), nnz);
        rowptr_from_hyper(dh.ptr, dp.ptr, nvec, A->nrows, d.p.ptr);
        d.j.alloc(nnz);
        narrow_u64(dc.ptr, d.j.ptr, nnz);
        if (A->valued()) { d.x.alloc(nnz); h2d(d.x.ptr, h.hval.data(), nnz); }
        sync_stream(); // host vectors are pageable: make sure staging copies are done before they can change
    }
    A->dev = std::move(d);
    A->dev_valid = true;
}

void ensure_dev(GrB_Matrix A) {
    finish_pending(A);
    if (A->dev_valid) return;
    if (A->bits_valid) {
        natural_bits(A);
        DevCSR d;
        bits_to_csr(A->bits, d);
        A->dev = std::move(d);
        if (A->valued()) { A->dev.x.alloc(A->dev.nnz); fill_u64(A->dev.x.ptr, 1, A->dev.nnz); }
        A->dev_valid = true;
        return;
    }
    upload_to_dev(A);
}

static void download_to_host(GrB_Matrix A) {
    if (A->host_valid) return;
    if (!A->dev_valid) ensure_dev(A);
    const DevCSR &d = A->dev;
    HostStore h;
    h.clear();
    if (d.nnz) {
        DevBuf<u64> dh, dp, dc(d.nnz);
        u64 nvec = hyper_from_rowptr(d.p.ptr, d.nrows, d.nnz, dh, dp);
        widen_u32(d.j.ptr, dc.ptr, d.nnz);
        h.hrow.resize(nvec);
        h.hptr.resize(nvec + 1);
        h.hcol.resize(d.nnz);
        d2h(h.hrow.data(), dh.ptr, nvec);
        d2h(h.hptr.data(), dp.ptr, nvec + 1);
        d2h(h.hcol.data(), dc.ptr, d.nnz);
        if (A->valued()) { h.hval.resize(d.nnz); d2h(h.hval.data(), d.x.ptr, d.nnz); }
        sync_stream();
    }
    A->host = std::move(h);
    A->host_valid = true;
}

void ensure_host(GrB_Matrix A) {
    if (!A->host_valid) download_to_host(A);
    finish_pending(A);
}

void ensure_bits(GrB_Matrix A) {
    finish_pending(A);
    if (A->bits_valid) { natural_bits(A); return; }
    ensure_dev(A);
    DevBits b;
    bits_from_csr(A->dev, b);
    A->bits = std::move(b);
    A->bits_nv = A->dev.nnz;
    A->bits_valid = true;
}

void ensure_devT(GrB_Matrix A) {
    ensure_dev(A);
    if (!A->devT_valid) {
        DevCSR t;
        transpose_csr(A->dev, t, false); // pattern-only mirror
        A->devT = std::move(t);
        A->devT_valid = true;
    }
    // pull-direction auxiliaries (hot-set packing, CSR-stream form, long-row lists) are built lazily by bits_hop
}

u64 matrix_nvals(GrB_Matrix A) {
    finish_pending(A);
    if (A->host_valid) return A->host.nnz();
    if (A->dev_valid) return A->dev.nnz;
    if (A->bits_nv == ~0ULL) A->bits_nv = bits_nvals(A->bits);   // popcount pass, remembered until the bit-matrix changes
    return A->bits_nv;
}

// ------------------------------------------------------------------------------------------------ write-back
static Desc get_desc(GrB_Descriptor d) {
    Desc r;
    if (d) { r.t0 = d->t0; r.t1 = d->t1; r.comp = d->comp; r.structure = d->structure; r.replace = d->replace; }
    return r;
}

// C<M,desc> = accum ? (C (+) T) : T       (GraphBLAS C API 2.1 write-back; accum is ANY or absent)
static void write_back(GrB_Matrix C, DevCSR &&T, GrB_Matrix M, const Desc &d, bool accum) {
    bool valued = C->valued();
    DevCSR Z;
    if (accum) {
        ensure_dev(C);
        ewise_union(C->dev, T, valued, Z);
    } else {
        Z = std::move(T);
    }
    if (!M) {
        if (d.comp) { // complement of "no mask" admits nothing
            if (d.replace) set_empty(C);
            return;
        }
        set_dev(C, std::move(Z));
        return;
    }
    ensure_dev(M);
    DevCSR Zm;
    filter_by_mask(Z, M->dev, d.comp, d.structure, Zm);
    if (d.replace) { set_dev(C, std::move(Zm)); return; }
    ensure_dev(C);
    DevCSR Ck, U;
    filter_by_mask(C->dev, M->dev, !d.comp, d.structure, Ck);
    ewise_union(Ck, Zm, valued, U);
    set_dev(C, std::move(U));
}

// ------------------------------------------------------------------------------------------------ host-resident matrices
// Matrices with a dimension >= 2^32 cannot be indexed by the device kernels (u32 column ids, dense rowptr).  The only
// such matrix on the path is Tensor's multi-edge store `me` (2^60 x 2^60, hypersparse, a handful of entries per
// multi-edge pair: tensor.rs:154-163, 254).  Its delta folds (VersionedMatrix::flush on `me`) still arrive as
// eWiseAdd / eWiseMult / masked-copy calls, so those three set operations exist on the hypersparse host form.  This is
// NOT a fallback: device-capable operands never take this branch (see is_huge), and mxm on such matrices is refused.
struct HTup { u64 r, c, v; };
bool is_huge(GrB_Matrix A) { return A && (A->nrows >= ((u64)1 << 32) || A->ncols >= ((u64)1 << 32)); }
static uvec<HTup> host_tuples(GrB_Matrix A) {
    ensure_host(A);
    const HostStore &h = A->host;
    uvec<HTup> t;
    t.reserve(h.nnz());
    for (u64 k = 0; k < h.hrow.size(); k++)
        for (u64 q = h.hptr[k]; q < h.hptr[k + 1]; q++) t.push_back(HTup{h.hrow[k], h.hcol[q], A->valued() ? h.hval[q] : 1});
    return t;
}
static inline bool tup_lt(const HTup &a, const HTup &b) { return a.r != b.r ? a.r < b.r : a.c < b.c; }
static inline bool tup_eq(const HTup &a, const HTup &b) { return a.r == b.r && a.c == b.c; }
static void host_store_from(GrB_Matrix C, const uvec<HTup> &t) {
    HostStore h;
    h.hptr.clear();
    for (const HTup &x : t) {
        if (h.hrow.empty() || h.hrow.back() != x.r) { h.hrow.push_back(x.r); h.hptr.push_back(h.hcol.size()); }
        h.hcol.push_back(x.c);
        if (C->valued()) h.hval.push_back(x.v);
    }
    h.hptr.push_back(h.hcol.size());
    set_empty(C);
    C->host = std::move(h);
}
static uvec<HTup> host_union(const uvec<HTup> &A, const uvec<HTup> &B) { // overlap: B's value
    uvec<HTup> o;
    o.reserve(A.size() + B.size());
    size_t i = 0, j = 0;
    while (i < A.size() || j < B.size()) {
        if (j >= B.size() || (i < A.size() && tup_lt(A[i], B[j]))) o.push_back(A[i++]);
        else if (i >= A.size() || tup_lt(B[j], A[i])) o.push_back(B[j++]);
        else { o.push_back(B[j]); i++; j++; }
    }
    return o;
}
static uvec<HTup> host_intersect(const uvec<HTup> &A, const uvec<HTup> &B) {
    uvec<HTup> o;
    size_t i = 0, j = 0;
    while (i < A.size() && j < B.size()) {
        if (tup_lt(A[i], B[j])) i++;
        else if (tup_lt(B[j], A[i])) j++;
        else { o.push_back(HTup{A[i].r, A[i].c, 1}); i++; j++; }
    }
    return o;
}
static uvec<HTup> host_filter(const uvec<HTup> &T, const uvec<HTup> &M, bool comp, bool structural, bool mvalued) {
    uvec<HTup> o;
    size_t j = 0;
    for (const HTup &x : T) {
        while (j < M.size() && tup_lt(M[j], x)) j++;
        bool in = j < M.size() && tup_eq(M[j], x) && (structural || !mvalued || M[j].v != 0);
        if (in != comp) o.push_back(x);
    }
    return o;
}
static void host_write_back(GrB_Matrix C, uvec<HTup> T, GrB_Matrix M, const Desc &d, bool accum) {
    uvec<HTup> Z = accum ? host_union(host_tuples(C), T) : std::move(T);
    if (!M) {
        if (d.comp) { if (d.replace) set_empty(C); return; }
        host_store_from(C, Z);
        return;
    }
    uvec<HTup> Mt = host_tuples(M);
    uvec<HTup> Zm = host_filter(Z, Mt, d.comp, d.structure, M->valued());
    if (d.replace) { host_store_from(C, Zm); return; }
    uvec<HTup> Ck = host_filter(host_tuples(C), Mt, !d.comp, d.structure, M->valued());
    host_store_from(C, host_union(Ck, Zm));
}

static void check_mask_dims(GrB_Matrix C, GrB_Matrix M) {
    if (M && (M->nrows != C->nrows || M->ncols != C->ncols)) throw GrbError(GrB_DIMENSION_MISMATCH, "mask dimensions differ from C");
}

// ================================================================================================ C ABI
extern "C" {

const char *B200_last_error(void) { return tl_error.c_str(); }

GrB_Info GxB_init(int mode, void *(*um)(size_t), void *(*uc)(size_t, size_t), void *(*ur)(void *, size_t), void (*uf)(void *)) {
    (void)mode;
    // Must precede every other call (as in the reference: matrix.rs:123-131 runs once at module load): memory obtained
    // from one allocator is never released with another.  malloc + free are mandatory (GraphBLAS C API: calloc / realloc may
    // be NULL and are then emulated).
    if (um && uf) {
        if (g_host_bytes.load() != 0) { tl_error = "GxB_init: allocator change with live host objects"; return GrB_INVALID_VALUE; }
        g_user_malloc = um; g_user_free = uf;
        g_user_calloc = uc; g_user_realloc = ur;
    }
    return GrB_SUCCESS; // the CUDA context is created lazily by the first bulk operation
}
GrB_Info GrB_init(int mode) { return GxB_init(mode, nullptr, nullptr, nullptr, nullptr); }
GrB_Info GrB_finalize(void) { return GrB_SUCCESS; }
GrB_Info GrB_Global_set_INT32(GrB_Global, int32_t, int field) {
    if (field == GxB_JIT_C_CONTROL || field == GxB_BURBLE) return GrB_SUCCESS;
    return GrB_INVALID_VALUE;
}
GrB_Info GxB_Global_Option_set_INT32(int field, int32_t) {
    if (field == GxB_NTHREADS) return GrB_SUCCESS; // host thread count is irrelevant to the GPU path
    return GrB_INVALID_VALUE;
}

// ---------------------------------------------------------------------------------------------- objects
GrB_Info GrB_Matrix_new(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols) {
    CHECK_PTR(A); CHECK_PTR(type);
    if (nrows > ((u64)1 << 60) || ncols > ((u64)1 << 60)) { tl_error = "dimension > 2^60"; return GrB_INVALID_VALUE; }
    return guarded([&]() {
        std::unique_ptr<GB_Matrix_opaque> mh(new GB_Matrix_opaque());   // released to the caller only on success
        GrB_Matrix m = mh.get();
        m->type = type->code;
        m->nrows = nrows; m->ncols = ncols;
        *A = mh.release();
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_free(GrB_Matrix *A) {
    if (!A || !*A) return GrB_SUCCESS;
    if ((*A)->magic != MAGIC) return GrB_INVALID_OBJECT;
    return guarded([&]() {
        GpuLock g;
        (*A)->magic = 0;
        delete *A;
        *A = nullptr;
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_dup(GrB_Matrix *C, GrB_Matrix A) {
    CHECK_PTR(C); CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        std::unique_ptr<GB_Matrix_opaque> mh(new GB_Matrix_opaque());   // released to the caller only on success
        GrB_Matrix m = mh.get();
        m->type = A->type; m->nrows = A->nrows; m->ncols = A->ncols;
        m->sparsity_control = A->sparsity_control; m->orientation = A->orientation;
        // pending work is copied, not finished (GB_dup; relied on by Matrix::grown, matrix.rs:691-698)
        m->pending = A->pending;
        m->host_valid = A->host_valid;
        if (A->host_valid) m->host = A->host;
        if (A->dev_valid) { csr_copy(A->dev, m->dev, true); m->dev_valid = true; }
        if (A->bits_valid && !A->dev_valid) { bits_copy(A->bits, m->bits); m->bits_valid = true; m->bits_nv = A->bits_nv; }
        *C = mh.release();
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_clear(GrB_Matrix A) {
    CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        set_empty(A);
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_resize(GrB_Matrix C, GrB_Index nr, GrB_Index nc) {
    CHECK_MAT(C);
    if (nr > ((u64)1 << 60) || nc > ((u64)1 << 60)) return GrB_INVALID_VALUE;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C};
        bool shrink = nr < C->nrows || nc < C->ncols;
        finish_pending(C);
        if (C->host_valid) {
            if (shrink) {
                HostStore &h = C->host, out;
                out.hptr.clear();
                bool valued = C->valued();
                for (u64 k = 0; k < h.hrow.size(); k++) {
                    if (h.hrow[k] >= nr) break;
                    size_t before = out.hcol.size();
                    for (u64 q = h.hptr[k]; q < h.hptr[k + 1]; q++) {
                        if (h.hcol[q] >= nc) break;
                        out.hcol.push_back(h.hcol[q]);
                        if (valued) out.hval.push_back(h.hval[q]);
                    }
                    if (out.hcol.size() > before) { out.hrow.push_back(h.hrow[k]); out.hptr.push_back(before); }
                }
                out.hptr.push_back(out.hcol.size());
                C->host = std::move(out);
            }
            C->nrows = nr; C->ncols = nc;
            C->dev_valid = false; C->dev.clear();
            C->bits_valid = false; C->bits.clear();
            invalidate_aux(C);
            return GrB_SUCCESS;
        }
        ensure_dev(C);
        if (nr >= ((u64)1 << 32) || nc >= ((u64)1 << 32)) { // leaves the device-capable range
            download_to_host(C);
            C->nrows = nr; C->ncols = nc;
            C->dev_valid = false; C->dev.clear();
            C->bits_valid = false; C->bits.clear();
            invalidate_aux(C);
            return GrB_SUCCESS;
        }
        DevCSR out;
        csr_resize(C->dev, nr, nc, out);
        C->nrows = nr; C->ncols = nc;
        set_dev(C, std::move(out));
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_nrows(GrB_Index *n, GrB_Matrix A) { CHECK_PTR(n); CHECK_MAT(A); *n = A->nrows; return GrB_SUCCESS; }
GrB_Info GrB_Matrix_ncols(GrB_Index *n, GrB_Matrix A) { CHECK_PTR(n); CHECK_MAT(A); *n = A->ncols; return GrB_SUCCESS; }
GrB_Info GrB_Matrix_nvals(GrB_Index *n, GrB_Matrix A) {
    CHECK_PTR(n); CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        *n = matrix_nvals(A);
        return GrB_SUCCESS;
    });
}

static u64 nonempty_rows(GrB_Matrix A) { return A->host.hrow.size(); }

GrB_Info GrB_Matrix_set_INT32(GrB_Matrix A, int32_t value, int field) {
    CHECK_MAT(A);
    switch (field) {
    case GxB_SPARSITY_CONTROL: A->sparsity_control = value; return GrB_SUCCESS;
    case GrB_STORAGE_ORIENTATION_HINT: A->orientation = value; return GrB_SUCCESS;
    case GxB_HYPER_HASH: A->hyper_hash = value; return GrB_SUCCESS;
    default: return GrB_INVALID_VALUE;
    }
}

GrB_Info GrB_Matrix_get_INT32(GrB_Matrix A, int32_t *value, int field) {
    CHECK_MAT(A); CHECK_PTR(value);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        switch (field) {
        case GxB_SPARSITY_CONTROL: *value = A->sparsity_control; return GrB_SUCCESS;
        case GrB_STORAGE_ORIENTATION_HINT: *value = A->orientation; return GrB_SUCCESS;
        case GxB_HYPER_HASH: *value = A->hyper_hash; return GrB_SUCCESS;
        case GxB_WILL_WAIT: *value = (!A->pending.empty() || (A->bits_valid && !A->dev_valid && !A->host_valid)) ? 1 : 0; return GrB_SUCCESS;
        case GxB_SPARSITY_STATUS: {
            // never bitmap/full on this path (matrix.rs:401-426, 558-575).  Hypersparse when pinned so,
            // or when allowed and fewer than 1/16 of the rows are non-empty (SuiteSparse hyper_switch).
            bool hyper = false;
            if (A->sparsity_control == GxB_HYPERSPARSE) hyper = true;
            else if ((A->sparsity_control & GxB_HYPERSPARSE) && A->host_valid && A->pending.empty()) {
                hyper = A->nrows > 1 && nonempty_rows(A) * 16 < A->nrows;
            }
            if (!(A->sparsity_control & GxB_SPARSE) && (A->sparsity_control & GxB_HYPERSPARSE)) hyper = true;
            *value = hyper ? GxB_HYPERSPARSE : GxB_SPARSE;
            return GrB_SUCCESS;
        }
        default: return GrB_INVALID_VALUE;
        }
    });
}

GrB_Info GxB_Matrix_type(GrB_Type *type, GrB_Matrix A) {
    CHECK_PTR(type); CHECK_MAT(A);
    *type = A->type == T_BOOL ? GrB_BOOL : A->type == T_UINT64 ? GrB_UINT64 : A->type == T_FP64 ? GrB_FP64 : GrB_INT64;
    return GrB_SUCCESS;
}
GrB_Info GxB_Matrix_iso(bool *iso, GrB_Matrix A) { CHECK_PTR(iso); CHECK_MAT(A); *iso = (A->type == T_BOOL); return GrB_SUCCESS; }
GrB_Info GxB_Matrix_memoryUsage(size_t *size, GrB_Matrix A) {
    CHECK_PTR(size); CHECK_MAT(A);
    size_t s = sizeof(GB_Matrix_opaque);
    s += (A->host.hrow.size() + A->host.hptr.size() + A->host.hcol.size() + A->host.hval.size()) * 8;
    s += A->pending.size() * sizeof(PendingOp);
    s += A->dev.p.bytes() + A->dev.j.bytes() + A->dev.x.bytes() + A->bits.w.bytes();
    s += A->devT.p.bytes() + A->devT.j.bytes() + A->devT.x.bytes();
    *size = s;
    return GrB_SUCCESS;
}
GrB_Info GxB_Matrix_fprint(GrB_Matrix A, const char *name, int pr, FILE *f) {
    CHECK_MAT(A);
    if (pr <= 0) return GrB_SUCCESS;
    if (!f) f = stdout;
    fprintf(f, "b200grb matrix %s: %llu x %llu, type %d, forms host=%d dev=%d bits=%d pending=%zu\n", name ? name : "",
            (unsigned long long)A->nrows, (unsigned long long)A->ncols, A->type, A->host_valid, A->dev_valid, A->bits_valid,
            A->pending.size());
    return GrB_SUCCESS;
}

GrB_Info GrB_Matrix_wait(GrB_Matrix A, int waitmode) {
    CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        finish_pending(A);
        if (waitmode == GrB_MATERIALIZE && !A->host_valid && !A->dev_valid && A->bits_valid) ensure_dev(A);
        if (A->dev_valid || A->bits_valid) sync_stream();
        return GrB_SUCCESS;
    });
}

// ---------------------------------------------------------------------------------------------- element access
static GrB_Info set_element(GrB_Matrix C, u64 v, u64 i, u64 j) {
    if (i >= C->nrows || j >= C->ncols) { tl_error = "setElement index out of bounds"; return GrB_INVALID_INDEX; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C};
        if (!C->host_valid) download_to_host(C);
        PendingOp op{i, j, v, (u64)C->pending.size(), false};
        C->pending.push_back(op);
        return GrB_SUCCESS;
    });
}
GrB_Info GrB_Matrix_setElement_BOOL(GrB_Matrix C, bool x, GrB_Index i, GrB_Index j) {
    CHECK_MAT(C);
    if (C->type == T_BOOL && !x) {
        tl_error = "BOOL matrices are pattern-only on this backend (stored false is never used on the path: versioned_matrix.rs:413-416)";
        return GrB_NOT_IMPLEMENTED;
    }
    return set_element(C, x ? 1 : 0, i, j);
}
GrB_Info GrB_Matrix_setElement_UINT64(GrB_Matrix C, uint64_t x, GrB_Index i, GrB_Index j) {
    CHECK_MAT(C);
    if (C->type == T_BOOL && x == 0) { tl_error = "typecast of 0 into a pattern-only BOOL matrix"; return GrB_NOT_IMPLEMENTED; }
    return set_element(C, C->type == T_BOOL ? 1 : x, i, j);
}
GrB_Info GrB_Matrix_removeElement(GrB_Matrix C, GrB_Index i, GrB_Index j) {
    CHECK_MAT(C);
    if (i >= C->nrows || j >= C->ncols) return GrB_INVALID_INDEX;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C};
        if (!C->host_valid) download_to_host(C);
        PendingOp op{i, j, 0, (u64)C->pending.size(), true};
        C->pending.push_back(op);
        return GrB_SUCCESS;
    });
}

// returns entry position or ~0
static u64 host_find(const HostStore &h, u64 i, u64 j) {
    auto it = std::lower_bound(h.hrow.begin(), h.hrow.end(), i);
    if (it == h.hrow.end() || *it != i) return ~0ULL;
    u64 k = (u64)(it - h.hrow.begin());
    auto b = h.hcol.begin() + h.hptr[k], e = h.hcol.begin() + h.hptr[k + 1];
    auto c = std::lower_bound(b, e, j);
    if (c == e || *c != j) return ~0ULL;
    return (u64)(c - h.hcol.begin());
}

static GrB_Info extract_element(u64 *x, GrB_Matrix A, u64 i, u64 j) {
    if (i >= A->nrows || j >= A->ncols) return GrB_INVALID_INDEX;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        if (!A->host_valid || !A->pending.empty()) ensure_host(A);
        u64 q = host_find(A->host, i, j);
        if (q == ~0ULL) return GrB_NO_VALUE;
        if (x) *x = A->valued() ? A->host.hval[q] : 1;
        return GrB_SUCCESS;
    });
}
GrB_Info GrB_Matrix_extractElement_BOOL(bool *x, GrB_Matrix A, GrB_Index i, GrB_Index j) {
    CHECK_MAT(A); CHECK_PTR(x);
    u64 v = 0;
    GrB_Info r = extract_element(&v, A, i, j);
    if (r == GrB_SUCCESS) *x = (v != 0);
    return r;
}
GrB_Info GrB_Matrix_extractElement_UINT64(uint64_t *x, GrB_Matrix A, GrB_Index i, GrB_Index j) {
    CHECK_MAT(A); CHECK_PTR(x);
    return extract_element(x, A, i, j);
}
GrB_Info GxB_Matrix_isStoredElement(GrB_Matrix A, GrB_Index i, GrB_Index j) {
    CHECK_MAT(A);
    return extract_element(nullptr, A, i, j);
}

static GrB_Info extract_tuples(GrB_Index *I, GrB_Index *J, void *X, int xkind, GrB_Index *nvals, GrB_Matrix A) {
    CHECK_MAT(A); CHECK_PTR(nvals);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_host(A);
        const HostStore &h = A->host;
        if (*nvals < h.nnz()) { tl_error = "extractTuples: output arrays too small"; return GrB_INSUFFICIENT_SPACE; }
        for (u64 k = 0; k < h.hrow.size(); k++)
            for (u64 q = h.hptr[k]; q < h.hptr[k + 1]; q++) {
                if (I) I[q] = h.hrow[k];
                if (J) J[q] = h.hcol[q];
                if (X) {
                    u64 v = A->valued() ? h.hval[q] : 1;
                    if (xkind == 1) ((bool *)X)[q] = v != 0; else ((uint64_t *)X)[q] = v;
                }
            }
        *nvals = h.nnz();
        return GrB_SUCCESS;
    });
}
GrB_Info GrB_Matrix_extractTuples_BOOL(GrB_Index *I, GrB_Index *J, bool *X, GrB_Index *nvals, GrB_Matrix A) {
    return extract_tuples(I, J, X, 1, nvals, A);
}
GrB_Info GrB_Matrix_extractTuples_UINT64(GrB_Index *I, GrB_Index *J, uint64_t *X, GrB_Index *nvals, GrB_Matrix A) {
    return extract_tuples(I, J, X, 2, nvals, A);
}

// ---------------------------------------------------------------------------------------------- build
GrB_Info GrB_Scalar_new(GrB_Scalar *s, GrB_Type type) {
    CHECK_PTR(s); CHECK_PTR(type);
    *s = new GB_Scalar_opaque{type->code, false, 0};
    return GrB_SUCCESS;
}
GrB_Info GrB_Scalar_setElement_BOOL(GrB_Scalar s, bool x) { CHECK_PTR(s); s->has = true; s->val = x ? 1 : 0; return GrB_SUCCESS; }
GrB_Info GrB_Scalar_free(GrB_Scalar *s) { if (s && *s) { delete *s; *s = nullptr; } return GrB_SUCCESS; }

static bool matrix_is_empty(GrB_Matrix C) {
    if (!C->pending.empty()) return false;
    if (C->host_valid) return C->host.nnz() == 0;
    if (C->dev_valid) return C->dev.nnz == 0;
    return bits_nvals(C->bits) == 0;
}

// host-side build for matrices outside the device-capable range (e.g. Tensor's 2^60 x 2^60 `me`)
static GrB_Info build_host(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const u64 *X, u64 n) {
    struct T { u64 i, j, v, s; };
    uvec<T> t(n);
    for (u64 k = 0; k < n; k++) {
        if (I[k] >= C->nrows || J[k] >= C->ncols) { tl_error = "build: index out of bounds"; return GrB_INDEX_OUT_OF_BOUNDS; }
        t[k] = T{I[k], J[k], X ? X[k] : 1, k};
    }
    std::sort(t.begin(), t.end(), [](const T &a, const T &b) {
        if (a.i != b.i) return a.i < b.i;
        if (a.j != b.j) return a.j < b.j;
        return a.s < b.s;
    });
    HostStore h;
    h.hptr.clear();
    for (u64 k = 0; k < n; k++) {
        if (k && t[k].i == t[k - 1].i && t[k].j == t[k - 1].j) continue;
        if (h.hrow.empty() || h.hrow.back() != t[k].i) { h.hrow.push_back(t[k].i); h.hptr.push_back(h.hcol.size()); }
        h.hcol.push_back(t[k].j);
        if (C->valued()) h.hval.push_back(t[k].v);
    }
    h.hptr.push_back(h.hcol.size());
    set_empty(C);
    C->host = std::move(h);
    return GrB_SUCCESS;
}

static GrB_Info build_common(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const u64 *X, u64 n) {
    CHECK_MAT(C);
    if (n) { CHECK_PTR(I); CHECK_PTR(J); }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C};
        if (!matrix_is_empty(C)) { tl_error = "build: output matrix not empty"; return GrB_OUTPUT_NOT_EMPTY; }
        if (n == 0) return GrB_SUCCESS;
        if (C->nrows >= ((u64)1 << 32) || C->ncols >= ((u64)1 << 32)) return build_host(C, I, J, X, n);
        ensure_init();
        DevBuf<u64> dI(n), dJ(n), dX;
        h2d(dI.ptr, (const u64 *)I, n);
        h2d(dJ.ptr, (const u64 *)J, n);
        if (X && C->valued()) { dX.alloc(n); h2d(dX.ptr, X, n); }
        DevCSR out;
        bool err = false;
        build_from_device_coo(dI.ptr, dJ.ptr, dX.ptr, n, C->nrows, C->ncols, out, &err);
        sync_stream();
        if (err) { tl_error = "build: index out of bounds"; return GrB_INDEX_OUT_OF_BOUNDS; }
        set_dev(C, std::move(out));
        return GrB_SUCCESS;
    });
}

GrB_Info GxB_Matrix_build_Scalar(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, GrB_Scalar scalar, GrB_Index nvals) {
    CHECK_PTR(scalar);
    if (!scalar->has) { tl_error = "build_Scalar: empty scalar"; return GrB_EMPTY_OBJECT; }
    if (C && C->magic == MAGIC && C->type == T_BOOL && scalar->val == 0) {
        tl_error = "build_Scalar(false) into a pattern-only BOOL matrix"; return GrB_NOT_IMPLEMENTED;
    }
    if (C && C->magic == MAGIC && C->valued()) {
        uvec<u64> X(nvals, scalar->val);
        return build_common(C, I, J, X.data(), nvals);
    }
    return build_common(C, I, J, nullptr, nvals);
}
GrB_Info GrB_Matrix_build_UINT64(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const uint64_t *X, GrB_Index nvals,
                                 GrB_BinaryOp dup) {
    (void)dup; // ANY (or any dup): the first tuple of a duplicate run wins, deterministically
    if (nvals) CHECK_PTR(X);
    if (C && C->magic == MAGIC && C->type == T_BOOL) {
        for (u64 k = 0; k < nvals; k++) if (X[k] == 0) { tl_error = "typecast of 0 into pattern-only BOOL"; return GrB_NOT_IMPLEMENTED; }
        return build_common(C, I, J, nullptr, nvals);
    }
    return build_common(C, I, J, X, nvals);
}
GrB_Info GrB_Matrix_build_BOOL(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const bool *X, GrB_Index nvals,
                               GrB_BinaryOp dup) {
    (void)dup;
    if (nvals) CHECK_PTR(X);
    CHECK_MAT(C);
    if (C->type == T_BOOL) {
        for (u64 k = 0; k < nvals; k++) if (!X[k]) { tl_error = "stored false in pattern-only BOOL"; return GrB_NOT_IMPLEMENTED; }
        return build_common(C, I, J, nullptr, nvals);
    }
    uvec<u64> V(nvals);
    for (u64 k = 0; k < nvals; k++) V[k] = X[k] ? 1 : 0;
    return build_common(C, I, J, V.data(), nvals);
}

// FP64 matrices (weighted paths: GrB_PLUS_TIMES_SEMIRING_FP64): values are stored as their IEEE-754 bit patterns
GrB_Info GrB_Matrix_build_FP64(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const double *X, GrB_Index nvals, GrB_BinaryOp dup) {
    (void)dup;   // duplicates: the first tuple of a run wins (GxB_ANY-like, deterministic); the reference builds from distinct edges
    if (nvals) CHECK_PTR(X);
    CHECK_MAT(C);
    if (C->type != T_FP64) { tl_error = "build_FP64 into a non-FP64 matrix"; return GrB_DOMAIN_MISMATCH; }
    static_assert(sizeof(double) == sizeof(u64), "FP64 travels in the u64 value arrays");
    return build_common(C, I, J, reinterpret_cast<const u64 *>(X), nvals);
}
GrB_Info GrB_Matrix_extractTuples_FP64(GrB_Index *I, GrB_Index *J, double *X, GrB_Index *nvals, GrB_Matrix A) {
    CHECK_MAT(A);
    if (A->type != T_FP64) {     // typecast from the integer / pattern types
        CHECK_PTR(nvals);
        uvec<u64> V(X ? *nvals : 0);
        GrB_Info r = extract_tuples(I, J, X ? V.data() : nullptr, 2, nvals, A);
        if (r == GrB_SUCCESS && X) for (u64 k = 0; k < *nvals; k++) X[k] = A->type == T_INT64 ? (double)(i64)V[k] : (double)V[k];
        return r;
    }
    return extract_tuples(I, J, X, 2, nvals, A);      // the stored bit patterns ARE the doubles
}

// ---------------------------------------------------------------------------------------------- mxm
static bool bits_legal(GrB_Matrix C, GrB_Matrix M, GrB_Matrix A, GrB_Matrix B, const Desc &d) {
    if (C->type != T_BOOL) return false;
    if (bits_words_for(A->nrows) == 0) return false;
    if (A->ncols >= ((u64)1 << 32) || B->ncols >= ((u64)1 << 32)) return false;
    if (M && !(d.comp && d.structure && d.replace)) return false; // the delta_lmxm form (matrix.rs:1383-1394)
    if (!M && d.comp) return false;
    return true;
}

// Y = A*B through the frontier dispatch: the push straight from A's entries while A is still a small CSR, the diagonal filter, or
// the direction-optimising push / pull.  pt_ok: the CSR push may write Y in B's hot-set order.  Returns true when Y came from
// A's CSR form (A then has no bit form).  acc (union hops): Y |= A*B into a natural-order Y that holds earlier operands' products.
extern "C++" bool frontier_product(GrB_Matrix A, GrB_Matrix B, bool pt_ok, DevBits &Y, u64 *fl, int *path, bool acc) {
    Context &cx = ctx();
    ensure_dev(B);
    if (B->diag_state < 0) B->diag_state = csr_is_diagonal(B->dev) ? 1 : 0;   // cached until B changes
    // a frontier that is still a (small) CSR expands straight from its entries unless it touches enough of B that the pull
    // should take it (only worth probing for a small CSR: the probe is O(nnz(F)))
    const bool from_csr = cx.opt_csr_push && A->dev_valid && !A->bits_valid && cx.opt_pull_mode != 1 &&
                          A->dev.nnz <= ((u64)1 << 20) &&
                          !(B->diag_state == 1 && cx.opt_diag_filter) &&
                          bits_push_from_csr(A->dev, B->dev, Y, fl, (B->devT_valid && pt_ok) ? &B->pt : (const PullTables *)nullptr, acc);
    if (from_csr) { *path = 7; return true; }
    if (!(A->bits_valid && A->pending.empty())) ensure_bits(A);   // an existing frontier keeps its vertex order for the hop
    if (B->diag_state == 1 && cx.opt_diag_filter) {
        natural_bits(A);
        if (acc) { DevBits Z; bits_diag(A->bits, B->dev, Z, fl); bits_or(Y, Z); }   // a diagonal type: a column filter, then OR
        else bits_diag(A->bits, B->dev, Y, fl);
        *path = 5;
    } else {
        if (cx.opt_pull_mode != 0) ensure_devT(B);
        bits_hop(A->bits, B->dev, B->devT_valid ? &B->devT : nullptr, B->devT_valid ? &B->pt : (PullTables *)nullptr, Y, fl, path, acc);
    }
    return false;
}

// The frontier bit-matrix path of GrB_mxm (short-fat A, CondTraverse's F*A): C<!M, RSC> = A*B kept in device frontier form.
// Returns false when the path does not apply (not legal, switched off, or the automatic choice prefers the general row-wise
// path); C is then unchanged.  dm / dp (B200_Matrix_delta_lmxm): device-resident deltas of B whose terms are applied to the
// product before it replaces C, while A's frontier is still intact: C = (A*B AND NOT A*dm) OR A*dp.
extern "C++" bool frontier_mxm(GrB_Matrix C, GrB_Matrix Mask, GrB_Matrix A, GrB_Matrix B, const Desc &d, bool accum,
                               const DevCSR *dm, const DevCSR *dp) {
    Context &cx = ctx();
    if (accum || d.t0 || d.t1 || cx.opt_bits_mode == 0 || !bits_legal(C, Mask, A, B, d)) return false;
    bool use_bits = (cx.opt_bits_mode == 1);
    finish_pending(A);
    if (!use_bits) {
        if (A->bits_valid && !A->dev_valid && !A->host_valid) use_bits = true; // stay in frontier form mid-chain
        else {
            ensure_dev(A); ensure_dev(B);
            use_bits = spgemm_flops(A->dev, B->dev) >= (u64)cx.opt_bits_min_flops;
        }
    }
    if (!use_bits) return false;
    DevBits Y;
    u64 fl = 0;
    int path = 0;
    const bool from_csr = frontier_product(A, B, !Mask, Y, &fl, &path);
    if (Mask) {
        ensure_bits(Mask);
        bits_andnot(Y, Mask->bits);
    }
    if (dm || dp) fl += bits_apply_deltas(from_csr ? nullptr : &A->bits, from_csr ? &A->dev : nullptr, dm, dp, Y);
    cx.last_flops = fl; cx.total_flops += fl; cx.last_path = (u64)path;
    set_bits(C, std::move(Y));
    if (cx.opt_sync_after_op) sync_stream();
    return true;
}

GrB_Info GrB_mxm(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Matrix A, GrB_Matrix B,
                 GrB_Descriptor desc) {
    CHECK_MAT(C); CHECK_MAT(A); CHECK_MAT(B); CHECK_PTR(semiring);
    if (Mask) CHECK_MAT(Mask);
    if (semiring != GxB_ANY_PAIR_BOOL) { tl_error = "mxm: only GxB_ANY_PAIR_BOOL is on the traversal path"; return GrB_NOT_IMPLEMENTED; }
    if (accum && accum != GxB_ANY_BOOL) { tl_error = "mxm: accum must be NULL or GxB_ANY_BOOL"; return GrB_NOT_IMPLEMENTED; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C, Mask, A, B};
        ensure_init();
        Context &cx = ctx();
        Desc d = get_desc(desc);
        u64 ar = d.t0 ? A->ncols : A->nrows, ac = d.t0 ? A->nrows : A->ncols;
        u64 br = d.t1 ? B->ncols : B->nrows, bc = d.t1 ? B->nrows : B->ncols;
        if (ac != br || C->nrows != ar || C->ncols != bc) throw GrbError(GrB_DIMENSION_MISMATCH, "mxm: dimension mismatch");
        check_mask_dims(C, Mask);

        // ---- frontier bit-matrix path (short-fat A, CondTraverse's F*A) ----
        if (frontier_mxm(C, Mask, A, B, d, accum != nullptr)) return GrB_SUCCESS;

        // ---- general row-wise path ----
        ensure_dev(A); ensure_dev(B);
        const DevCSR *Ad = &A->dev, *Bd = &B->dev;
        if (d.t0) { ensure_devT(A); Ad = &A->devT; }
        if (d.t1) { ensure_devT(B); Bd = &B->devT; }
        if (Mask && !d.comp && !accum) {
            // C<M> = A*B: fused -- the product is only ever evaluated at M's positions (matrix-level ExpandInto)
            ensure_dev(Mask);
            u64 fl = spgemm_flops(*Ad, *Bd);
            DevCSR Zm;
            spgemm_masked(*Ad, *Bd, Mask->dev, d.structure, Zm, fl);
            cx.last_flops = fl; cx.total_flops += fl; cx.last_path = 6;
            if (d.replace) set_dev(C, std::move(Zm));
            else {
                ensure_dev(C);
                DevCSR Ck, U;
                filter_by_mask(C->dev, Mask->dev, true, d.structure, Ck);
                ewise_union(Ck, Zm, C->valued(), U);
                set_dev(C, std::move(U));
            }
            if (cx.opt_sync_after_op) sync_stream();
            return GrB_SUCCESS;
        }
        DevCSR T;
        u64 fl = 0;
        spgemm_anypair(*Ad, *Bd, T, &fl);
        cx.last_flops = fl; cx.total_flops += fl; cx.last_path = 1;
        write_back(C, std::move(T), Mask, d, accum != nullptr);
        if (cx.opt_sync_after_op) sync_stream();
        return GrB_SUCCESS;
    });
}

// ---------------------------------------------------------------------------------------------- eWise / transpose / apply
static void check_same_dims(GrB_Matrix C, u64 r, u64 c, const char *what) {
    if (C->nrows != r || C->ncols != c) throw GrbError(GrB_DIMENSION_MISMATCH, std::string(what) + ": dimension mismatch");
}
static const DevCSR *operand(GrB_Matrix A, bool transposed) {
    ensure_dev(A);
    if (!transposed) return &A->dev;
    ensure_devT(A);
    return &A->devT;
}

GrB_Info GrB_Matrix_eWiseAdd_BinaryOp(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_BinaryOp add, GrB_Matrix A,
                                      GrB_Matrix B, GrB_Descriptor desc) {
    CHECK_MAT(C); CHECK_MAT(A); CHECK_MAT(B); CHECK_PTR(add);
    if (Mask) CHECK_MAT(Mask);
    if (accum) { tl_error = "eWiseAdd: accum not on the path"; return GrB_NOT_IMPLEMENTED; }
    if (add != GxB_ANY_BOOL && add != GrB_SECOND_UINT64 && add != GxB_ANY_UINT64) {
        tl_error = "eWiseAdd: op must be GxB_ANY_BOOL / GrB_SECOND_UINT64 / GxB_ANY_UINT64"; return GrB_NOT_IMPLEMENTED;
    }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C, Mask, A, B};
        if (!is_huge(C) && !is_huge(A)) ensure_init();   // host-resident operands need no device
        Desc d = get_desc(desc);
        u64 ar = d.t0 ? A->ncols : A->nrows, ac = d.t0 ? A->nrows : A->ncols;
        u64 br = d.t1 ? B->ncols : B->nrows, bc = d.t1 ? B->nrows : B->ncols;
        if (ar != br || ac != bc) throw GrbError(GrB_DIMENSION_MISMATCH, "eWiseAdd: operand dimensions differ");
        check_same_dims(C, ar, ac, "eWiseAdd");
        check_mask_dims(C, Mask);
        if (!C->valued() && (A->valued() || B->valued()))
            throw GrbError(GrB_NOT_IMPLEMENTED, "eWiseAdd: valued -> BOOL typecast is not on the path (use apply(ONE): matrix.rs:898-905)");
        if (is_huge(C)) {   // Tensor.me delta fold
            if (d.t0 || d.t1) throw GrbError(GrB_NOT_IMPLEMENTED, "eWiseAdd: transposed operands on a host-resident matrix");
            host_write_back(C, host_union(host_tuples(A), host_tuples(B)), Mask, d, false);
            return GrB_SUCCESS;
        }
        // frontier form: C = A u B with no mask is a word-wise OR (delta_lmxm's accum step, matrix.rs:1398-1400)
        if (!Mask && !d.comp && !d.t0 && !d.t1 && !C->valued() && (A->bits_valid || B->bits_valid) &&
            A->pending.empty() && B->pending.empty() && bits_words_for(A->nrows) != 0 &&
            ((A->bits_valid && !A->dev_valid && !A->host_valid) || (B->bits_valid && !B->dev_valid && !B->host_valid))) {
            ensure_bits(A); ensure_bits(B);
            DevBits Y;
            natural_bits(A); natural_bits(B);
            bits_copy(A->bits, Y);
            bits_or(Y, B->bits);
            set_bits(C, std::move(Y));
            return GrB_SUCCESS;
        }
        if (C->valued() && (d.t0 || d.t1))
            throw GrbError(GrB_NOT_IMPLEMENTED, "eWiseAdd: transposed valued operands are not on the path");
        const DevCSR *Ad = operand(A, d.t0), *Bd = operand(B, d.t1);
        DevCSR T;
        ewise_union(*Ad, *Bd, C->valued(), T);
        write_back(C, std::move(T), Mask, d, false);
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_eWiseMult_Semiring(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_Semiring semiring,
                                       GrB_Matrix A, GrB_Matrix B, GrB_Descriptor desc) {
    CHECK_MAT(C); CHECK_MAT(A); CHECK_MAT(B); CHECK_PTR(semiring);
    if (Mask) CHECK_MAT(Mask);
    if (accum) { tl_error = "eWiseMult: accum not on the path"; return GrB_NOT_IMPLEMENTED; }
    if (semiring != GxB_ANY_PAIR_BOOL) { tl_error = "eWiseMult: only GxB_ANY_PAIR_BOOL"; return GrB_NOT_IMPLEMENTED; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C, Mask, A, B};
        if (!is_huge(C) && !is_huge(A)) ensure_init();   // host-resident operands need no device
        Desc d = get_desc(desc);
        u64 ar = d.t0 ? A->ncols : A->nrows, ac = d.t0 ? A->nrows : A->ncols;
        u64 br = d.t1 ? B->ncols : B->nrows, bc = d.t1 ? B->nrows : B->ncols;
        if (ar != br || ac != bc) throw GrbError(GrB_DIMENSION_MISMATCH, "eWiseMult: operand dimensions differ");
        check_same_dims(C, ar, ac, "eWiseMult");
        check_mask_dims(C, Mask);
        if (is_huge(C)) {
            if (d.t0 || d.t1) throw GrbError(GrB_NOT_IMPLEMENTED, "eWiseMult: transposed operands on a host-resident matrix");
            host_write_back(C, host_intersect(host_tuples(A), host_tuples(B)), Mask, d, false);
            return GrB_SUCCESS;
        }
        const DevCSR *Ad = operand(A, d.t0), *Bd = operand(B, d.t1);
        DevCSR T;
        ewise_intersect(*Ad, *Bd, T);
        write_back(C, std::move(T), Mask, d, false);
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_transpose(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_Matrix A, GrB_Descriptor desc) {
    CHECK_MAT(C); CHECK_MAT(A);
    if (Mask) CHECK_MAT(Mask);
    if (accum) { tl_error = "transpose: accum not on the path"; return GrB_NOT_IMPLEMENTED; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C, Mask, A};
        if (!is_huge(C) && !is_huge(A)) ensure_init();   // host-resident operands need no device
        Desc d = get_desc(desc);
        // T = (A^T0)' : with T0 set the double transpose is the identity (masked copy, matrix.rs:824-845)
        bool eff_transpose = !d.t0;
        u64 tr = eff_transpose ? A->ncols : A->nrows, tc = eff_transpose ? A->nrows : A->ncols;
        check_same_dims(C, tr, tc, "transpose");
        check_mask_dims(C, Mask);
        if (!C->valued() && A->valued())
            throw GrbError(GrB_NOT_IMPLEMENTED, "transpose: valued -> BOOL typecast is not on the path");
        if (is_huge(C) || is_huge(A)) {
            uvec<HTup> T = host_tuples(A);
            if (eff_transpose) {
                for (HTup &x : T) std::swap(x.r, x.c);
                std::sort(T.begin(), T.end(), tup_lt);
            }
            if (!C->valued()) for (HTup &x : T) x.v = 1;
            host_write_back(C, std::move(T), Mask, d, false);
            return GrB_SUCCESS;
        }
        ensure_dev(A);
        DevCSR T;
        if (eff_transpose) transpose_csr(A->dev, T, C->valued());
        else csr_copy(A->dev, T, C->valued());
        write_back(C, std::move(T), Mask, d, false);
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Matrix_apply(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_UnaryOp op, GrB_Matrix A, GrB_Descriptor desc) {
    CHECK_MAT(C); CHECK_MAT(A); CHECK_PTR(op);
    if (Mask) CHECK_MAT(Mask);
    if (op != GxB_ONE_BOOL) { tl_error = "apply: only GxB_ONE_BOOL (set_pattern, matrix.rs:906-924)"; return GrB_NOT_IMPLEMENTED; }
    if (accum && accum != GxB_ANY_BOOL) { tl_error = "apply: accum must be NULL or GxB_ANY_BOOL"; return GrB_NOT_IMPLEMENTED; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{C, Mask, A};
        if (!is_huge(C) && !is_huge(A)) ensure_init();   // host-resident operands need no device
        Desc d = get_desc(desc);
        u64 ar = d.t0 ? A->ncols : A->nrows, ac = d.t0 ? A->nrows : A->ncols;
        check_same_dims(C, ar, ac, "apply");
        check_mask_dims(C, Mask);
        if (is_huge(C)) {
            if (d.t0) throw GrbError(GrB_NOT_IMPLEMENTED, "apply: transposed operand on a host-resident matrix");
            uvec<HTup> T = host_tuples(A);
            for (HTup &x : T) x.v = 1;
            host_write_back(C, std::move(T), Mask, d, accum != nullptr);
            return GrB_SUCCESS;
        }
        const DevCSR *Ad = operand(A, d.t0);
        DevCSR T;
        csr_copy(*Ad, T, false); // ONE: pattern of A, every value true -- A's values are never read
        write_back(C, std::move(T), Mask, d, accum != nullptr);
        return GrB_SUCCESS;
    });
}

// ---------------------------------------------------------------------------------------------- iterator
GrB_Info GxB_Iterator_new(GxB_Iterator *it) { CHECK_PTR(it); *it = new GB_Iterator_opaque(); return GrB_SUCCESS; }
GrB_Info GxB_Iterator_free(GxB_Iterator *it) { if (it && *it) { delete *it; *it = nullptr; } return GrB_SUCCESS; }

GrB_Info GxB_rowIterator_attach(GxB_Iterator it, GrB_Matrix A, GrB_Descriptor) {
    CHECK_PTR(it); CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        it->A = A; it->k = 0; it->q = 0; it->exhausted = true;
        it->bitmap = false; it->bm.clear(); it->bm.shrink_to_fit();
        if (A->pending.empty() && !A->host_valid && A->bits_valid && A->bits.nrows == A->nrows && !A->valued() && !is_huge(A)) {
            ensure_init();
            natural_bits(A);
            const u64 nv = A->dev_valid ? A->dev.nnz : bits_nvals(A->bits);
            if (A->nrows && A->ncols && nv > (A->nrows * A->ncols) / 32) {   // denser than one entry per 32 slots
                const u64 wpr = (A->ncols + 63) / 64;
                it->bm.resize(A->nrows * wpr);
                DevBuf<u64> stage(A->nrows * wpr);
                bits_to_rowmajor(A->bits, stage.ptr, wpr);
                d2h(it->bm.data(), stage.ptr, A->nrows * wpr);
                sync_stream();
                it->bitmap = true; it->wpr = wpr; it->nrows = A->nrows; it->ncols = A->ncols;
                return GrB_SUCCESS;
            }
        }
        if (!A->host_valid || !A->pending.empty()) ensure_host(A);
        return GrB_SUCCESS;
    });
}
GrB_Index GxB_rowIterator_kount(GxB_Iterator it) {
    if (!it || !it->A) return 0;
    if (it->bitmap) return it->nrows;
    GrB_Matrix A = it->A;
    int32_t st = GxB_SPARSE;
    GrB_Matrix_get_INT32(A, &st, GxB_SPARSITY_STATUS);
    return st == GxB_HYPERSPARSE ? (GrB_Index)A->host.hrow.size() : A->nrows;
}
// positions at the first stored row >= `row`; empty rows are skipped (hypersparse behaviour; the
// reference loops over GrB_NO_VALUE rows anyway, matrix.rs:1523-1531)
GrB_Info GxB_rowIterator_seekRow(GxB_Iterator it, GrB_Index row) {
    CHECK_PTR(it); CHECK_PTR(it->A);
    if (it->bitmap) {
        for (u64 r = row; r < it->nrows; r++) {
            u64 c = it->first_set(r, 0);
            if (c < it->ncols) { it->k = r; it->q = c; it->exhausted = false; return GrB_SUCCESS; }
        }
        it->exhausted = true;
        return GxB_EXHAUSTED;
    }
    const HostStore &h = it->A->host;
    u64 k = (u64)(std::lower_bound(h.hrow.begin(), h.hrow.end(), row) - h.hrow.begin());
    it->k = k;
    if (k >= h.hrow.size()) { it->exhausted = true; return GxB_EXHAUSTED; }
    it->q = h.hptr[k];
    it->exhausted = false;
    return GrB_SUCCESS;
}
GrB_Info GxB_rowIterator_nextRow(GxB_Iterator it) {
    CHECK_PTR(it); CHECK_PTR(it->A);
    if (it->bitmap) {
        if (it->exhausted) return GxB_EXHAUSTED;
        return GxB_rowIterator_seekRow(it, it->k + 1);
    }
    const HostStore &h = it->A->host;
    if (it->exhausted) return GxB_EXHAUSTED;
    it->k++;
    if (it->k >= h.hrow.size()) { it->exhausted = true; return GxB_EXHAUSTED; }
    it->q = h.hptr[it->k];
    return GrB_SUCCESS;
}
GrB_Info GxB_rowIterator_nextCol(GxB_Iterator it) {
    CHECK_PTR(it); CHECK_PTR(it->A);
    if (it->bitmap) {
        if (it->exhausted) return GxB_EXHAUSTED;
        u64 c = it->first_set(it->k, it->q + 1);
        if (c < it->ncols) { it->q = c; return GrB_SUCCESS; }
        return GrB_NO_VALUE;
    }
    const HostStore &h = it->A->host;
    if (it->exhausted) return GxB_EXHAUSTED;
    if (it->q + 1 < h.hptr[it->k + 1]) { it->q++; return GrB_SUCCESS; }
    return GrB_NO_VALUE; // end of this row; position unchanged
}
GrB_Index GxB_rowIterator_getRowIndex(GxB_Iterator it) {
    if (!it || !it->A) return 0;
    if (it->bitmap) return it->exhausted ? it->nrows : it->k;
    const HostStore &h = it->A->host;
    if (it->exhausted || it->k >= h.hrow.size()) return it->A->nrows; // SuiteSparse returns nrows when exhausted
    return h.hrow[it->k];
}
GrB_Index GxB_rowIterator_getColIndex(GxB_Iterator it) {
    if (!it || !it->A || it->exhausted) return 0;
    if (it->bitmap) return it->q;
    return it->A->host.hcol[it->q];
}
static u64 vec_at(GrB_Vector v, u64 k);
uint64_t GxB_Iterator_get_UINT64(GxB_Iterator it) {
    if (it && it->V) {
        if (it->exhausted) return 0;
        return it->V->full ? vec_at(it->V, it->k) : (uint64_t)it->V->val[it->k];
    }
    if (!it || !it->A || it->exhausted) return 0;
    if (it->bitmap) return 1;
    return it->A->valued() ? it->A->host.hval[it->q] : 1;
}
bool GxB_Iterator_get_BOOL(GxB_Iterator it) { return GxB_Iterator_get_UINT64(it) != 0; }

// ---------------------------------------------------------------------------------------------- vectors
GrB_Info GrB_Vector_new(GrB_Vector *v, GrB_Type type, GrB_Index n) {
    CHECK_PTR(v); CHECK_PTR(type);
    GrB_Vector x = new GB_Vector_opaque();
    x->type = type->code; x->n = n;
    *v = x;
    return GrB_SUCCESS;
}
GrB_Info GrB_Vector_free(GrB_Vector *v) { if (v && *v) { if ((*v)->fx) g_user_free((*v)->fx); delete *v; *v = nullptr; } return GrB_SUCCESS; }
GrB_Info GrB_Vector_size(GrB_Index *n, GrB_Vector v) { CHECK_PTR(n); CHECK_PTR(v); *n = v->n; return GrB_SUCCESS; }
GrB_Info GrB_Vector_nvals(GrB_Index *n, GrB_Vector v) { CHECK_PTR(n); CHECK_PTR(v); *n = v->full ? v->n : v->idx.size(); return GrB_SUCCESS; }
// a full (container payload) vector that is written element-wise drops back to the sparse form first
static void vec_make_sparse(GrB_Vector v);
static GrB_Info vec_set(GrB_Vector v, i64 x, GrB_Index i) {
    CHECK_PTR(v);
    if (i >= v->n) return GrB_INVALID_INDEX;
    return guarded([&]() {
        vec_make_sparse(v);
        if (v->idx.empty() || v->idx.back() < i) { v->idx.push_back(i); v->val.push_back(x); return GrB_SUCCESS; }   // ascending fill: O(1)
        auto it = std::lower_bound(v->idx.begin(), v->idx.end(), i);
        size_t pos = it - v->idx.begin();
        if (it != v->idx.end() && *it == i) v->val[pos] = x;
        else { v->idx.insert(it, i); v->val.insert(v->val.begin() + pos, x); }
        return GrB_SUCCESS;
    });
}
GrB_Info GrB_Vector_setElement_BOOL(GrB_Vector v, bool x, GrB_Index i) { return vec_set(v, x ? 1 : 0, i); }          // vector.rs:127, 507
GrB_Info GrB_Vector_setElement_UINT64(GrB_Vector v, uint64_t x, GrB_Index i) { return vec_set(v, (i64)x, i); }     // vector.rs:442
GrB_Info GrB_Vector_removeElement(GrB_Vector v, GrB_Index i) {                                                       // vector.rs:519
    CHECK_PTR(v);
    if (i >= v->n) return GrB_INVALID_INDEX;
    return guarded([&]() {
        vec_make_sparse(v);
        auto it = std::lower_bound(v->idx.begin(), v->idx.end(), i);
        if (it != v->idx.end() && *it == i) { v->val.erase(v->val.begin() + (it - v->idx.begin())); v->idx.erase(it); }
        return GrB_SUCCESS;            // removing an absent entry is not an error (GraphBLAS C API 2.1)
    });
}
GrB_Info GrB_Vector_clear(GrB_Vector v) {                                                                            // vector.rs:98
    CHECK_PTR(v);
    v->idx.clear(); v->val.clear();
    if (v->fx) { g_user_free(v->fx); v->fx = nullptr; }
    v->full = false; v->fbytes = 0;
    return GrB_SUCCESS;
}
GrB_Info GrB_Vector_wait(GrB_Vector v, int) { CHECK_PTR(v); return GrB_SUCCESS; }   // nothing is ever left pending (vector.rs:134)
GrB_Info GrB_Vector_resize(GrB_Vector v, GrB_Index n) {                                                              // vector.rs:494
    CHECK_PTR(v);
    return guarded([&]() {
        if (n < v->n) {
            vec_make_sparse(v);
            size_t keep = std::lower_bound(v->idx.begin(), v->idx.end(), n) - v->idx.begin();
            v->idx.resize(keep); v->val.resize(keep);
        } else if (n > v->n && v->full) vec_make_sparse(v);
        v->n = n;
        return GrB_SUCCESS;
    });
}
GrB_Info GrB_Vector_extractElement_INT64(int64_t *x, GrB_Vector v, GrB_Index i) {
    CHECK_PTR(x); CHECK_PTR(v);
    if (i >= v->n) return GrB_INVALID_INDEX;
    auto it = std::lower_bound(v->idx.begin(), v->idx.end(), i);
    if (it == v->idx.end() || *it != i) return GrB_NO_VALUE;
    *x = v->val[it - v->idx.begin()];
    return GrB_SUCCESS;
}
GrB_Info GrB_Vector_extractElement_BOOL(bool *x, GrB_Vector v, GrB_Index i) {
    int64_t t = 0;
    CHECK_PTR(x);
    GrB_Info r = GrB_Vector_extractElement_INT64(&t, v, i);
    if (r == GrB_SUCCESS) *x = t != 0;
    return r;
}
static u64 vec_at(GrB_Vector v, u64 k);
static inline double bits_as_double(i64 b) { double x; memcpy(&x, &b, 8); return x; }
GrB_Info GrB_Vector_extractTuples_INT64(GrB_Index *I, int64_t *X, GrB_Index *nvals, GrB_Vector v) {
    CHECK_PTR(nvals); CHECK_PTR(v);
    const u64 nv = v->full ? v->n : v->idx.size();
    if (*nvals < nv) return GrB_INSUFFICIENT_SPACE;
    for (u64 k = 0; k < nv; k++) {
        if (I) I[k] = v->full ? k : v->idx[k];
        if (X) X[k] = v->full ? (v->type == T_FP64 ? (int64_t)((const double *)v->fx)[k] : (int64_t)vec_at(v, k))
                              : (v->type == T_FP64 ? (int64_t)bits_as_double(v->val[k]) : v->val[k]);
    }
    *nvals = nv;
    return GrB_SUCCESS;
}
GrB_Info GrB_Vector_extractTuples_BOOL(GrB_Index *I, bool *X, GrB_Index *nvals, GrB_Vector v) {
    CHECK_PTR(nvals); CHECK_PTR(v);
    if (*nvals < v->idx.size()) return GrB_INSUFFICIENT_SPACE;
    for (size_t k = 0; k < v->idx.size(); k++) { if (I) I[k] = v->idx[k]; if (X) X[k] = v->val[k] != 0; }
    *nvals = v->idx.size();
    return GrB_SUCCESS;
}

// ---- vector iterator (vector.rs:553-594): positions 0 .. nvals-1 in ascending index order
static u64 vec_nvals(GrB_Vector v) { return v->full ? v->n : v->idx.size(); }
GrB_Info GxB_Vector_Iterator_attach(GxB_Iterator it, GrB_Vector v, GrB_Descriptor) {
    CHECK_PTR(it); CHECK_PTR(v);
    it->A = nullptr; it->bitmap = false; it->bm.clear();
    it->V = v; it->k = 0; it->q = 0;
    it->exhausted = vec_nvals(v) == 0;
    return GrB_SUCCESS;
}
GrB_Index GxB_Vector_Iterator_getpmax(GxB_Iterator it) { return (it && it->V) ? vec_nvals(it->V) : 0; }
GrB_Index GxB_Vector_Iterator_getp(GxB_Iterator it) { return (it && it->V) ? it->k : 0; }
GrB_Info GxB_Vector_Iterator_seek(GxB_Iterator it, GrB_Index p) {
    if (!it || !it->V) return GrB_NULL_POINTER;
    const u64 pmax = vec_nvals(it->V);
    if (p >= pmax) { it->k = pmax; it->exhausted = true; return GxB_EXHAUSTED; }
    it->k = p; it->exhausted = false;
    return GrB_SUCCESS;
}
GrB_Info GxB_Vector_Iterator_next(GxB_Iterator it) {
    if (!it || !it->V) return GrB_NULL_POINTER;
    const u64 pmax = vec_nvals(it->V);
    if (it->k + 1 >= pmax) { it->k = pmax; it->exhausted = true; return GxB_EXHAUSTED; }
    it->k++;
    return GrB_SUCCESS;
}
GrB_Index GxB_Vector_Iterator_getIndex(GxB_Iterator it) {
    if (!it || !it->V || it->exhausted) return 0;
    return it->V->full ? it->k : it->V->idx[it->k];
}

// ---- FP64 vectors (values as bit patterns in `val` / as doubles in a full payload) ----
static inline i64 f64_bits(double x) { i64 b; memcpy(&b, &x, 8); return b; }
static inline double bits_f64(i64 b) { double x; memcpy(&x, &b, 8); return x; }
static double vec_value_f64(GrB_Vector v, u64 k) {       // k-th stored entry as a double (typecast from the integer types)
    if (v->full) {
        if (v->type == T_FP64) return ((const double *)v->fx)[k];
        return v->type == T_INT64 ? (double)(i64)vec_at(v, k) : (double)vec_at(v, k);
    }
    if (v->type == T_FP64) return bits_f64(v->val[k]);
    return v->type == T_UINT64 ? (double)(u64)v->val[k] : (double)v->val[k];     // `val` is i64: UINT64 >= 2^63 must not turn negative
}
GrB_Info GrB_Vector_setElement_FP64(GrB_Vector v, double x, GrB_Index i) {
    CHECK_PTR(v);
    if (v->type != T_FP64) { tl_error = "setElement_FP64 into a non-FP64 vector"; return GrB_DOMAIN_MISMATCH; }
    return vec_set(v, f64_bits(x), i);
}
GrB_Info GrB_Vector_extractElement_FP64(double *x, GrB_Vector v, GrB_Index i) {
    CHECK_PTR(x); CHECK_PTR(v);
    if (i >= v->n) return GrB_INVALID_INDEX;
    if (v->full) { *x = vec_value_f64(v, i); return GrB_SUCCESS; }
    auto it = std::lower_bound(v->idx.begin(), v->idx.end(), i);
    if (it == v->idx.end() || *it != i) return GrB_NO_VALUE;
    *x = vec_value_f64(v, it - v->idx.begin());
    return GrB_SUCCESS;
}
// the call algo.pageRank reads its result through (algo_procedures.rs: extract_vector_f64)
GrB_Info GrB_Vector_extractTuples_FP64(GrB_Index *I, double *X, GrB_Index *nvals, GrB_Vector v) {
    CHECK_PTR(nvals); CHECK_PTR(v);
    const u64 nv = v->full ? v->n : v->idx.size();
    if (*nvals < nv) return GrB_INSUFFICIENT_SPACE;
    for (u64 k = 0; k < nv; k++) { if (I) I[k] = v->full ? k : v->idx[k]; if (X) X[k] = vec_value_f64(v, k); }
    *nvals = nv;
    return GrB_SUCCESS;
}

// w = A*u (mxv) or u*A (vxm) over PLUS_TIMES_FP64 / PLUS_SECOND_FP64: dense device vectors, sparse semantics kept through a
// presence byte per entry (w(i) exists iff some A(i,k) meets an existing u(k)).  accum: NULL or GrB_PLUS_FP64; no mask.
static GrB_Info mxv_fp64_entry(GrB_Vector w, GrB_Vector mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Vector u, GrB_Matrix A,
                               GrB_Descriptor desc, bool is_mxv) {
    CHECK_PTR(w); CHECK_PTR(u); CHECK_MAT(A);
    if (mask) { tl_error = "FP64 mxv/vxm: masks are not on this path"; return GrB_NOT_IMPLEMENTED; }
    if (accum && accum != GrB_PLUS_FP64) { tl_error = "FP64 mxv/vxm: accum must be NULL or GrB_PLUS_FP64"; return GrB_NOT_IMPLEMENTED; }
    if (w->type != T_FP64) { tl_error = "FP64 mxv/vxm: the output vector must be GrB_FP64"; return GrB_DOMAIN_MISMATCH; }
    const bool times = semiring->code == SR_PLUS_TIMES_FP64;
    if (times && A->type != T_FP64) { tl_error = "PLUS_TIMES_FP64 needs a GrB_FP64 matrix"; return GrB_DOMAIN_MISMATCH; }
    Desc d = get_desc(desc);
    const bool a_transposed = is_mxv ? d.t0 : !d.t1;          // rows of the operand we stream = output indices
    const u64 outer = a_transposed ? A->ncols : A->nrows, inner = a_transposed ? A->nrows : A->ncols;
    if (u->n != inner || w->n != outer) return GrB_DIMENSION_MISMATCH;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        const DevCSR *Ad = &A->dev;
        DevCSR T;
        if (a_transposed) {
            if (times) { transpose_csr(A->dev, T, true); Ad = &T; }      // valued transpose (the cached mirror is pattern-only)
            else { ensure_devT(A); Ad = &A->devT; }
        }
        // u -> dense
        uvec<double> hx(inner, 0.0);
        uvec<unsigned char> hp(inner, 0);
        const u64 unv = u->full ? u->n : u->idx.size();
        for (u64 k = 0; k < unv; k++) { const u64 i = u->full ? k : u->idx[k]; hx[i] = vec_value_f64(u, k); hp[i] = 1; }
        DevBuf<double> dx(inner ? inner : 1), dy(outer ? outer : 1);
        DevBuf<unsigned char> dp(inner ? inner : 1), dyp(outer ? outer : 1);
        h2d(dx.ptr, hx.data(), inner); h2d(dp.ptr, hp.data(), inner);
        uvec<double> hy(outer, 0.0);
        uvec<unsigned char> hw(outer, 0);
        if (accum) {
            const u64 wnv = w->full ? w->n : w->idx.size();
            for (u64 k = 0; k < wnv; k++) { const u64 i = w->full ? k : w->idx[k]; hy[i] = vec_value_f64(w, k); hw[i] = 1; }
            h2d(dy.ptr, hy.data(), outer);
        }
        mxv_fp64(*Ad, times, dx.ptr, unv == inner ? nullptr : dp.ptr, dy.ptr, dyp.ptr, 0.0, accum != nullptr);
        uvec<unsigned char> hyp(outer, 0);
        d2h(hy.data(), dy.ptr, outer); d2h(hyp.data(), dyp.ptr, outer);
        sync_stream();
        vec_make_sparse(w);
        w->idx.clear(); w->val.clear();
        for (u64 i = 0; i < outer; i++)
            if (hyp[i] || (accum && hw[i])) { w->idx.push_back(i); w->val.push_back(f64_bits(hy[i])); }
        return GrB_SUCCESS;
    });
}

// one frontier step w<mask> = u*A (vxm) or A*u (mxv) over ANY_PAIR, run as a 1-row mxm
static GrB_Info frontier_step(GrB_Vector w, GrB_Vector mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Vector u,
                              GrB_Matrix A, GrB_Descriptor desc, bool is_mxv) {
    CHECK_PTR(w); CHECK_PTR(u); CHECK_MAT(A);
    if (semiring != GxB_ANY_PAIR_BOOL || accum) { tl_error = "vxm/mxv: ANY_PAIR, no accum"; return GrB_NOT_IMPLEMENTED; }
    Desc d = get_desc(desc);
    // vxm: w' = u' * A (T1 transposes A).  mxv: w = A*u <=> w' = u' * A' (T0 transposes A).
    bool a_transposed = is_mxv ? !d.t0 : d.t1;
    u64 inner = a_transposed ? A->ncols : A->nrows, outer = a_transposed ? A->nrows : A->ncols;
    if (u->n != inner || w->n != outer || (mask && mask->n != outer)) return GrB_DIMENSION_MISMATCH;
    GrB_Matrix F = nullptr, Mm = nullptr, Cm = nullptr;
    GrB_Info info = GrB_Matrix_new(&F, GrB_BOOL, 1, inner);
    if (info) return info;
    GrB_Matrix_new(&Cm, GrB_BOOL, 1, outer);
    uvec<u64> zeros(std::max(u->idx.size(), mask ? mask->idx.size() : (size_t)0), 0);
    GrB_Scalar s; GrB_Scalar_new(&s, GrB_BOOL); GrB_Scalar_setElement_BOOL(s, true);
    uvec<u64> uidx;
    for (size_t k = 0; k < u->idx.size(); k++) if (u->val[k] != 0 || u->type != T_BOOL) uidx.push_back(u->idx[k]);
    info = GxB_Matrix_build_Scalar(F, zeros.data(), uidx.data(), s, uidx.size());
    if (!info && mask) {
        GrB_Matrix_new(&Mm, GrB_BOOL, 1, outer);
        uvec<u64> midx;
        for (size_t k = 0; k < mask->idx.size(); k++) if (d.structure || mask->val[k] != 0) midx.push_back(mask->idx[k]);
        info = GxB_Matrix_build_Scalar(Mm, zeros.data(), midx.data(), s, midx.size());
    }
    if (!info) {
        // existing w content matters only without replace; seed C with it
        if (mask && !d.replace && !w->idx.empty()) {
            uvec<u64> z2(w->idx.size(), 0);
            info = GxB_Matrix_build_Scalar(Cm, z2.data(), w->idx.data(), s, w->idx.size());
        }
    }
    if (!info) {
        GB_Descriptor_opaque dd = {false, a_transposed, d.comp, true, d.replace};
        info = GrB_mxm(Cm, Mm, nullptr, GxB_ANY_PAIR_BOOL, F, A, &dd);
    }
    if (!info) {
        GrB_Index nv = 0;
        GrB_Matrix_nvals(&nv, Cm);
        uvec<u64> I(nv), J(nv);
        GrB_Index cap = nv;
        info = GrB_Matrix_extractTuples_BOOL(I.data(), J.data(), nullptr, &cap, Cm);
        if (!info) {
            w->idx.assign(J.begin(), J.end());
            w->val.assign(nv, 1);
        }
    }
    GrB_Scalar_free(&s);
    GrB_Matrix_free(&F); GrB_Matrix_free(&Mm); GrB_Matrix_free(&Cm);
    return info;
}
GrB_Info GrB_vxm(GrB_Vector w, GrB_Vector mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Vector u, GrB_Matrix A,
                 GrB_Descriptor desc) {
    CHECK_PTR(semiring);
    if (semiring->code != SR_ANY_PAIR) return mxv_fp64_entry(w, mask, accum, semiring, u, A, desc, false);
    return frontier_step(w, mask, accum, semiring, u, A, desc, false);
}
GrB_Info GrB_mxv(GrB_Vector w, GrB_Vector mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Matrix A, GrB_Vector u,
                 GrB_Descriptor desc) {
    CHECK_PTR(semiring);
    if (semiring->code != SR_ANY_PAIR) return mxv_fp64_entry(w, mask, accum, semiring, u, A, desc, true);
    return frontier_step(w, mask, accum, semiring, u, A, desc, true);
}

// ---------------------------------------------------------------------------------------------- LAGraph subset
int LAGraph_Init(char *msg) { if (msg) msg[0] = 0; return 0; }
int LAGraph_Finalize(char *msg) { if (msg) msg[0] = 0; return 0; }
int LAGraph_New(LAGraph_Graph *G, GrB_Matrix *A, LAGraph_Kind kind, char *msg) {
    if (msg) msg[0] = 0;
    if (!G) return GrB_NULL_POINTER;
    LAGraph_Graph g = (LAGraph_Graph)calloc(1, sizeof(struct LAGraph_Graph_struct));
    if (!g) return GrB_OUT_OF_MEMORY;
    g->kind = kind;
    if (A) { g->A = *A; *A = nullptr; } // the matrix MOVES into the graph (lagraph_bindings.rs:175)
    g->is_symmetric_structure = -1; g->nself_edges = -1;
    *G = g;
    return 0;
}
int LAGraph_Delete(LAGraph_Graph *G, char *msg) {
    if (msg) msg[0] = 0;
    if (!G || !*G) return 0;
    GrB_Matrix_free(&(*G)->A);
    GrB_Matrix_free(&(*G)->AT);
    GrB_Vector_free(&(*G)->out_degree);
    GrB_Vector_free(&(*G)->in_degree);
    free(*G);
    *G = nullptr;
    return 0;
}

extern "C" GrB_Info B200_Matrix_prepare(GrB_Matrix A, int want_transpose);
// LAGraph's cached properties the reference asks for before PageRank (algo_procedures.rs:748-749): the transpose mirror lives
// inside the matrix handle here, out-degrees are read off A's row pointers -- both calls only make sure the mirror exists.
int LAGraph_Cached_AT(LAGraph_Graph G, char *msg) {
    if (msg) msg[0] = 0;
    if (!G || !G->A) return GrB_NULL_POINTER;
    return B200_Matrix_prepare(G->A, 1);
}
int LAGraph_Cached_OutDegree(LAGraph_Graph G, char *msg) {
    if (msg) msg[0] = 0;
    return (!G || !G->A) ? GrB_NULL_POINTER : GrB_SUCCESS;
}
// LAGr_PageRank (lagraph_bindings.rs:549-558; call site algo_procedures.rs:744-752).  Computed in FP64 on the device (algo.cu);
// centrality is a full GrB_FP64 vector, read by the reference through GrB_Vector_extractTuples_FP64.
int LAGr_PageRank(GrB_Vector *centrality, int *iters, LAGraph_Graph G, float damping, float tol, int itermax, char *msg) {
    if (msg) msg[0] = 0;
    if (!G || !G->A || !centrality || !iters) return GrB_NULL_POINTER;
    GrB_Matrix A = G->A;
    if (A->magic != MAGIC) return GrB_INVALID_OBJECT;
    if (A->nrows != A->ncols) return GrB_DIMENSION_MISMATCH;
    GrB_Info info = guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_devT(A);
        const u64 n = A->nrows;
        DevBuf<double> r(n ? n : 1);
        *iters = pagerank(A->dev, A->devT, (double)damping, (double)tol, itermax, r.ptr);
        std::unique_ptr<GB_Vector_opaque> v(new GB_Vector_opaque());
        v->type = T_FP64; v->n = n; v->full = true; v->fbytes = n * sizeof(double);
        if (n) {
            v->fx = g_user_malloc(v->fbytes);
            if (!v->fx) throw std::bad_alloc();
            CUDA_TRY(cudaMemcpyAsync(v->fx, r.ptr, v->fbytes, cudaMemcpyDeviceToHost, stream()));
            sync_stream();
        }
        *centrality = v.release();
        return GrB_SUCCESS;
    });
    if (info && msg) snprintf(msg, 256, "%s", tl_error.c_str());
    return info;
}
// LAGr_ConnectedComponents (lagraph_bindings.rs:521-526; call site algo_procedures.rs:838-846): component(i) = the smallest vertex
// id of i's component, a full (dense) GrB_UINT64 vector as LAGraph documents.  The pattern must be symmetric (the reference passes
// build_symmetric_adjacency_matrix and sets is_symmetric_structure); a directed graph is refused like LAGraph does (-1005).
int LAGr_ConnectedComponents(GrB_Vector *component, LAGraph_Graph G, char *msg) {
    if (msg) msg[0] = 0;
    if (!G || !G->A || !component) return GrB_NULL_POINTER;
    GrB_Matrix A = G->A;
    if (A->magic != MAGIC) return GrB_INVALID_OBJECT;
    if (A->nrows != A->ncols) return GrB_DIMENSION_MISMATCH;
    if (G->kind != LAGraph_ADJACENCY_UNDIRECTED && G->is_symmetric_structure != 1) {
        if (msg) snprintf(msg, 256, "G->A must be known to be symmetric");
        return -1005;       // LAGRAPH_SYMMETRIC_STRUCTURE_REQUIRED
    }
    GrB_Info info = guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        const u64 n = A->nrows;
        DevBuf<u64> comp(n ? n : 1);
        connected_components(A->dev, comp.ptr);
        std::unique_ptr<GB_Vector_opaque> v(new GB_Vector_opaque());
        v->type = T_UINT64; v->n = n; v->full = true; v->fbytes = n * sizeof(u64);
        if (n) {
            v->fx = g_user_malloc(v->fbytes);
            if (!v->fx) throw std::bad_alloc();
            CUDA_TRY(cudaMemcpyAsync(v->fx, comp.ptr, v->fbytes, cudaMemcpyDeviceToHost, stream()));
            sync_stream();
        }
        *component = v.release();
        return GrB_SUCCESS;
    });
    if (info && msg) snprintf(msg, 256, "%s", tl_error.c_str());
    return info;
}
// LAGraph_cdlp (lagraphx_bindings.rs:218-223; call site algo_procedures.rs:1232-1237): label(i) after at most `itermax` rounds of
// synchronous label propagation from label(i) = i, a full GrB_UINT64 vector.  The reference always passes the symmetric adjacency
// (build_symmetric_adjacency_matrix, kind UNDIRECTED), so "neighbours" are the entries of row i; a directed graph is refused.
int LAGraph_cdlp(GrB_Vector *CDLP_handle, LAGraph_Graph G, int itermax, char *msg) {
    if (msg) msg[0] = 0;
    if (!G || !G->A || !CDLP_handle) return GrB_NULL_POINTER;
    GrB_Matrix A = G->A;
    if (A->magic != MAGIC) return GrB_INVALID_OBJECT;
    if (A->nrows != A->ncols) return GrB_DIMENSION_MISMATCH;
    if (itermax < 0) return GrB_INVALID_VALUE;
    if (G->kind != LAGraph_ADJACENCY_UNDIRECTED && G->is_symmetric_structure != 1) {
        if (msg) snprintf(msg, 256, "G->A must be known to be symmetric");
        return -1005;       // LAGRAPH_SYMMETRIC_STRUCTURE_REQUIRED
    }
    GrB_Info info = guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        const u64 n = A->nrows;
        DevBuf<u64> lab(n ? n : 1);
        cdlp(A->dev, itermax, lab.ptr);
        std::unique_ptr<GB_Vector_opaque> v(new GB_Vector_opaque());
        v->type = T_UINT64; v->n = n; v->full = true; v->fbytes = n * sizeof(u64);
        if (n) {
            v->fx = g_user_malloc(v->fbytes);
            if (!v->fx) throw std::bad_alloc();
            CUDA_TRY(cudaMemcpyAsync(v->fx, lab.ptr, v->fbytes, cudaMemcpyDeviceToHost, stream()));
            sync_stream();
        }
        *CDLP_handle = v.release();
        return GrB_SUCCESS;
    });
    if (info && msg) snprintf(msg, 256, "%s", tl_error.c_str());
    return info;
}
// One BFS over rows [lo, lo + nrows(A)) of the n-vertex graph; level / parent of those rows go to `location` memory.  With AT
// (the same rows of A') the direction-optimising engine runs, its out-degree table cached on A; without it (one GPU, lo = 0)
// the top-down bfs_run.  Both give level and minimum-id parent.  dest >= 0 stops once that vertex is reached.  dirty (one GPU,
// B200_bfs_delta): the engine walks those operands instead of A, with deg / total_edges from bfs_delta_degrees.
extern "C++" void bfs_staged(GrB_Matrix A, const DevCSR *AT, u64 n, u64 lo, BfsComm *comm, u64 src, i64 max_level, i64 dest,
                             i64 *level, i64 *parent, int location, B200_BfsInfo *info_out,
                             const std::vector<BfsOperand> *dirty, const u32 *deg, u64 total_edges) {
    const u64 nloc = A->nrows, hi = lo + nloc;
    DevBuf<i64> dl, dp;
    i64 *d_level = level, *d_parent = parent;
    if (location != B200_LOC_DEVICE) {
        dl.alloc(nloc ? nloc : 1); d_level = dl.ptr;
        if (parent) { dp.alloc(nloc ? nloc : 1); d_parent = dp.ptr; }
    }
    BfsInfo rec;
    memset(&rec, 0, sizeof(rec));
    if (dirty) {
        bfs_do(A->dev, A->dev, n, lo, hi, deg, total_edges, comm, src, max_level, dest, d_level, d_parent, &rec, dirty);
    } else if (AT) {
        if (!A->bfs_deg_valid) { bfs_build_degrees(A->dev, n, lo, hi, comm, A->bfs_deg, &A->bfs_edges); A->bfs_deg_valid = true; }
        bfs_do(A->dev, *AT, n, lo, hi, A->bfs_deg.ptr, A->bfs_edges, comm, src, max_level, dest, d_level, d_parent, &rec);
    } else {
        if (dest >= 0) throw GrbError(GrB_NOT_IMPLEMENTED, "BFS with a destination needs the transpose mirror (B200_Matrix_prepare)");
        bfs_run(A->dev, src, max_level, d_level, d_parent, &rec.edges);
    }
    if (location != B200_LOC_DEVICE) {
        d2h(level, d_level, nloc);
        if (parent) d2h(parent, d_parent, nloc);
    }
    sync_stream();
    if (info_out) memcpy(info_out, &rec, sizeof(rec));
}
// Single-GPU BFS.  With the transpose mirror in place (B200_Matrix_prepare(A, 1), or any earlier pull) the direction-optimising
// engine runs; without it -- one BFS on a fresh matrix, where building A' would cost more than the search -- the top-down one.
GrB_Info B200_bfs_ex(GrB_Matrix A, GrB_Index src, int64_t max_level, int64_t dest, int64_t *level, int64_t *parent, int location,
                     B200_BfsInfo *info_out) {
    CHECK_MAT(A); CHECK_PTR(level);
    if (A->nrows != A->ncols) { tl_error = "BFS needs a square adjacency matrix"; return GrB_DIMENSION_MISMATCH; }
    if (src >= A->nrows || (dest >= 0 && (u64)dest >= A->nrows)) return GrB_INVALID_INDEX;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        bfs_staged(A, A->devT_valid ? &A->devT : nullptr, A->nrows, 0, nullptr, src, max_level, dest, level, parent, location, info_out);
        return GrB_SUCCESS;
    });
}
GrB_Info B200_bfs(GrB_Matrix A, GrB_Index src, int64_t max_level, int64_t *level, int64_t *parent, int location,
                  uint64_t *edges_traversed) {
    B200_BfsInfo info;
    memset(&info, 0, sizeof(info));
    GrB_Info r = B200_bfs_ex(A, src, max_level, -1, level, parent, location, &info);
    if (r == GrB_SUCCESS && edges_traversed) *edges_traversed = info.edges;
    return r;
}

// ---- NCCL communicator of the partitioned BFS: rank 0 creates the id, the caller ships its 128 bytes to the other ranks by
// whatever means it has (the tests and bench.py: torch.distributed broadcast), every rank then calls B200_comm_init ----
GrB_Info B200_comm_unique_id(uint8_t *id128) {
    CHECK_PTR(id128);
    return guarded([&]() { ensure_init(); comm_unique_id(id128); return GrB_SUCCESS; });
}
GrB_Info B200_comm_init(B200_Comm *comm, int rank, int world, const uint8_t *id128) {
    CHECK_PTR(comm);
    if (world > 1) CHECK_PTR(id128);
    return guarded([&]() { GpuLock g; ensure_init(); *comm = (B200_Comm)comm_init(rank, world, id128); return GrB_SUCCESS; });
}
GrB_Info B200_comm_free(B200_Comm *comm) {
    if (!comm || !*comm) return GrB_SUCCESS;
    return guarded([&]() { GpuLock g; sync_stream(); comm_free((BfsComm *)*comm); *comm = nullptr; return GrB_SUCCESS; });
}
// 1-D row-block partitioned BFS (BASELINE config 5): Alocal = rows [row_lo, row_lo + nrows(Alocal)) of the n x n adjacency
// matrix, ATlocal = the same rows of its transpose (both with global column ids); row blocks are ceil(n / P) rounded up to 64.
// level_local / parent_local: int64[nrows(Alocal)] (host or device by `location`).  Collective: every rank calls it.
GrB_Info B200_bfs_partitioned(GrB_Matrix Alocal, GrB_Matrix ATlocal, uint64_t n, uint64_t row_lo, B200_Comm comm, GrB_Index src,
                              int64_t max_level, int64_t dest, int64_t *level_local, int64_t *parent_local, int location,
                              B200_BfsInfo *info_out) {
    CHECK_MAT(Alocal); CHECK_MAT(ATlocal); CHECK_PTR(level_local);
    if (Alocal->ncols != n || ATlocal->ncols != n || Alocal->nrows != ATlocal->nrows || row_lo + Alocal->nrows > n) {
        tl_error = "partitioned BFS: Alocal / ATlocal must be (hi - lo) x n row blocks"; return GrB_DIMENSION_MISMATCH;
    }
    if (src >= n || (dest >= 0 && (u64)dest >= n)) return GrB_INVALID_INDEX;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{Alocal, ATlocal};
        ensure_init();
        ensure_dev(Alocal); ensure_dev(ATlocal);
        bfs_staged(Alocal, &ATlocal->dev, n, row_lo, (BfsComm *)comm, src, max_level, dest, level_local, parent_local, location, info_out);
        return GrB_SUCCESS;
    });
}

int LAGr_BreadthFirstSearch_Extended(GrB_Vector *level, GrB_Vector *parent, LAGraph_Graph G, GrB_Index src, int64_t max_level,
                                     int64_t dest, bool many_expected, char *msg) {
    (void)many_expected;
    if (msg) msg[0] = 0;
    if (!G || !G->A) return GrB_NULL_POINTER;
    if (dest >= 0) {   // early exit at `dest` (lagraphx_bindings.rs:585-594) runs on the direction-optimising engine: needs A' (LAGraph's cached AT)
        GrB_Info pi = B200_Matrix_prepare(G->A, 1);
        if (pi) { if (msg) snprintf(msg, 256, "%s", tl_error.c_str()); return pi; }
    }
    u64 n = G->A->nrows;
    uvec<i64> lv(n), pr;
    if (parent) pr.resize(n);
    GrB_Info info = B200_bfs_ex(G->A, src, max_level < 0 ? -1 : max_level, dest, lv.data(), parent ? pr.data() : nullptr, B200_LOC_HOST, nullptr);
    if (info) { if (msg) snprintf(msg, 256, "%s", tl_error.c_str()); return info; }
    auto fill = [&](GrB_Vector *out, const uvec<i64> &src_v) {
        GrB_Vector v = new GB_Vector_opaque();
        v->type = T_INT64; v->n = n;
        for (u64 i = 0; i < n; i++) if (src_v[i] >= 0) { v->idx.push_back(i); v->val.push_back(src_v[i]); }
        *out = v;
    };
    if (level) fill(level, lv);
    if (parent) fill(parent, pr);
    return 0;
}

// ---------------------------------------------------------------------------------------------- B200 extensions
GrB_Info B200_Matrix_import_CSR(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols, const uint64_t *Ap,
                                const uint32_t *Aj, const uint64_t *Ax, int location) {
    CHECK_PTR(A); CHECK_PTR(type); CHECK_PTR(Ap);
    if (nrows >= ((u64)1 << 32) || ncols >= ((u64)1 << 32)) return GrB_NOT_IMPLEMENTED;
    return guarded([&]() {
        GpuLock g;
        ensure_init();
        std::unique_ptr<GB_Matrix_opaque> mh(new GB_Matrix_opaque());   // released to the caller only on success
        GrB_Matrix m = mh.get();
        m->type = type->code; m->nrows = nrows; m->ncols = ncols;
        DevCSR d;
        d.nrows = nrows; d.ncols = ncols;
        d.p.alloc(nrows + 1);
        u64 nnz;
        if (location == B200_LOC_DEVICE) {
            d2d(d.p.ptr, (const u64 *)Ap, nrows + 1);
            nnz = read_scalar(d.p.ptr + nrows);
        } else {
            nnz = Ap[nrows];
            h2d(d.p.ptr, (const u64 *)Ap, nrows + 1);
        }
        d.nnz = nnz;
        d.j.alloc(nnz);
        bool vals = m->valued() && Ax;
        if (vals) d.x.alloc(nnz);
        if (location == B200_LOC_DEVICE) { d2d(d.j.ptr, (const u32 *)Aj, nnz); if (vals) d2d(d.x.ptr, (const u64 *)Ax, nnz); }
        else { h2d(d.j.ptr, (const u32 *)Aj, nnz); if (vals) h2d(d.x.ptr, (const u64 *)Ax, nnz); }
        sync_stream();
        set_dev(m, std::move(d));
        *A = mh.release();
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_export_CSR(GrB_Matrix A, uint64_t *Ap, uint32_t *Aj, uint64_t *Ax, int location) {
    CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        const DevCSR &d = A->dev;
        if (location == B200_LOC_DEVICE) {
            if (Ap) d2d((u64 *)Ap, d.p.ptr, d.nrows + 1);
            if (Aj) d2d((u32 *)Aj, d.j.ptr, d.nnz);
            if (Ax && d.has_values()) d2d((u64 *)Ax, d.x.ptr, d.nnz);
        } else {
            if (Ap) d2h((u64 *)Ap, d.p.ptr, d.nrows + 1);
            if (Aj) d2h((u32 *)Aj, d.j.ptr, d.nnz);
            if (Ax && d.has_values()) d2h((u64 *)Ax, d.x.ptr, d.nnz);
        }
        sync_stream();
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_export_bitmap(GrB_Matrix A, uint64_t *bits_out, uint64_t words_per_row, uint64_t *nvals_out, int location) {
    CHECK_MAT(A);
    if (!bits_out) { tl_error = "export_bitmap: null output"; return GrB_NULL_POINTER; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        finish_pending(A);
        const u64 wpr = (A->ncols + 63) / 64;
        if (words_per_row != wpr) throw GrbError(GrB_DIMENSION_MISMATCH, "export_bitmap: words_per_row must be ceil(ncols / 64)");
        if (A->nrows && wpr > (1ULL << 36) / A->nrows) throw GrbError(GrB_OUT_OF_MEMORY, "export_bitmap: bitmap larger than 512 GiB");
        const u64 total = A->nrows * wpr;
        const bool from_bits = A->bits_valid && A->bits.nrows == A->nrows;
        if (!from_bits) ensure_dev(A); else natural_bits(A);
        DevBuf<u64> stage;
        u64 *dst = (u64 *)bits_out;
        if (location != B200_LOC_DEVICE) { stage.alloc(total); dst = stage.ptr; }
        if (from_bits) {
            bits_to_rowmajor(A->bits, dst, wpr);
            if (nvals_out) { if (A->bits_nv == ~0ULL) A->bits_nv = bits_nvals(A->bits); *nvals_out = A->bits_nv; }
        } else {
            if (total) CUDA_TRY(cudaMemsetAsync(dst, 0, total * sizeof(u64), stream()));
            csr_to_rowmajor(A->dev, dst, wpr);
            if (nvals_out) *nvals_out = A->dev.nnz;
        }
        if (location != B200_LOC_DEVICE && total) d2h((u64 *)bits_out, dst, total);
        sync_stream();
        return GrB_SUCCESS;
    });
}

// ---- asynchronous bitmap hand-off: the D2H copy runs on a second stream, so the next batch's hops overlap it ----
struct B200_Ticket_opaque {
    DevBuf<u64> stage;          // row-major bitmap on the device, alive until the copy has finished
    cudaEvent_t done = nullptr; // recorded on the copy stream after the D2H
};
static cudaStream_t g_copy_stream = nullptr;

GrB_Info B200_Matrix_export_bitmap_async(GrB_Matrix A, uint64_t *bits_out, uint64_t words_per_row, B200_Ticket *ticket) {
    CHECK_MAT(A);
    if (!bits_out || !ticket) { tl_error = "export_bitmap_async: null argument"; return GrB_NULL_POINTER; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        finish_pending(A);
        const u64 wpr = (A->ncols + 63) / 64;
        if (words_per_row != wpr) throw GrbError(GrB_DIMENSION_MISMATCH, "export_bitmap_async: words_per_row must be ceil(ncols / 64)");
        if (A->nrows && wpr > (1ULL << 36) / A->nrows) throw GrbError(GrB_OUT_OF_MEMORY, "export_bitmap_async: bitmap larger than 512 GiB");
        const u64 total = A->nrows * wpr;
        const bool from_bits = A->bits_valid && A->bits.nrows == A->nrows;
        if (!from_bits) ensure_dev(A); else natural_bits(A);
        if (!g_copy_stream) CUDA_TRY(cudaStreamCreateWithFlags(&g_copy_stream, cudaStreamNonBlocking));
        std::unique_ptr<B200_Ticket_opaque> t(new B200_Ticket_opaque());
        t->stage.alloc(total);
        if (from_bits) bits_to_rowmajor(A->bits, t->stage.ptr, wpr);
        else {
            if (total) CUDA_TRY(cudaMemsetAsync(t->stage.ptr, 0, total * sizeof(u64), stream()));
            csr_to_rowmajor(A->dev, t->stage.ptr, wpr);
        }
        // from here on the copy stream may be reading the stage: on any failure drain it before the stage returns to the
        // (single-stream) pool, and release both events
        struct Ev { cudaEvent_t e = nullptr; ~Ev() { if (e) cudaEventDestroy(e); } } ready, done;
        try {
            CUDA_TRY(cudaEventCreateWithFlags(&ready.e, cudaEventDisableTiming));
            CUDA_TRY(cudaEventRecord(ready.e, stream()));
            CUDA_TRY(cudaStreamWaitEvent(g_copy_stream, ready.e, 0));
            if (total) {
                // asynchronous only for page-locked bits_out; a pageable destination makes this call block until the copy is done
                CUDA_TRY(cudaMemcpyAsync(bits_out, t->stage.ptr, total * sizeof(u64), cudaMemcpyDeviceToHost, g_copy_stream));
                ctx().d2h_bytes += total * sizeof(u64);
            }
            CUDA_TRY(cudaEventCreateWithFlags(&done.e, cudaEventDisableTiming));
            CUDA_TRY(cudaEventRecord(done.e, g_copy_stream));
        } catch (...) {
            cudaStreamSynchronize(g_copy_stream);
            throw;
        }
        t->done = done.e;
        done.e = nullptr;
        *ticket = t.release();
        return GrB_SUCCESS;
    });
}
// blocks until the copy behind `ticket` has landed in the caller's buffer, then releases the ticket
GrB_Info B200_Ticket_wait(B200_Ticket *ticket) {
    if (!ticket || !*ticket) return GrB_SUCCESS;
    return guarded([&]() {
        B200_Ticket t = *ticket;
        *ticket = nullptr;
        cudaError_t e = cudaEventSynchronize(t->done);
        cudaEventDestroy(t->done);
        {
            GpuLock g;     // the staging block goes back to the (single-stream) pool
            t->stage.release();
        }
        delete t;
        if (e != cudaSuccess) throw CudaError(e, __FILE__, __LINE__);
        return GrB_SUCCESS;
    });
}

// Order-sensitive digest of A's pattern in CSR order (materialises A on the device first): the full-size parity tests compare
// multi-GB results through these three numbers against the oracle's digest of its own result (oracle/grb_oracle.c: orc_digest).
GrB_Info B200_Matrix_digest(GrB_Matrix A, uint64_t *digest3) {
    CHECK_MAT(A); CHECK_PTR(digest3);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        if (is_huge(A)) throw GrbError(GrB_NOT_IMPLEMENTED, "digest: host-resident matrix");
        ensure_dev(A);
        csr_digest(A->dev, digest3);
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_device_view(GrB_Matrix A, const uint64_t **Ap, const uint32_t **Aj, const uint64_t **Ax) {
    CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        sync_stream();
        if (Ap) *Ap = A->dev.p.ptr;
        if (Aj) *Aj = A->dev.j.ptr;
        if (Ax) *Ax = A->dev.x.ptr;
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_prepare(GrB_Matrix A, int want_transpose) {
    CHECK_MAT(A);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        if (want_transpose) {
            ensure_devT(A);
            bits_prepare_pull(A->dev, A->devT, A->pt);     // hot-set order, relabelled col_idx, segment list: off the first query's path
        }
        sync_stream();
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_push_operand(GrB_Matrix A, uint32_t *ap_out, uint32_t *pperm_out, int *sorted) {
    CHECK_MAT(A);
    CHECK_PTR(sorted);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        if (!A->devT_valid || !A->pt.ap.ptr || !A->pt.pperm) throw GrbError(GrB_INVALID_VALUE, "push_operand: the matrix has no relabelled col_idx (not prepared, or not square)");
        if (ap_out) d2h(ap_out, A->pt.ap.ptr, A->pt.ap.n);
        if (pperm_out) d2h(pperm_out, A->pt.pperm->ptr, A->pt.pperm->n);
        sync_stream();
        *sorted = A->pt.ap_sorted ? 1 : 0;
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_rmat(GrB_Matrix *A, int scale, uint64_t edge_factor, uint64_t seed) {
    CHECK_PTR(A);
    return guarded([&]() {
        GpuLock g;
        ensure_init();
        std::unique_ptr<GB_Matrix_opaque> mh(new GB_Matrix_opaque());   // released to the caller only on success
        GrB_Matrix m = mh.get();
        if (scale < 1 || scale > 31) throw GrbError(GrB_INVALID_VALUE, "rmat: scale must be in [1, 31]");
        m->type = T_BOOL; m->nrows = m->ncols = (u64)1 << scale;
        DevCSR d;
        rmat_csr(scale, edge_factor, seed, d);
        sync_stream();
        set_dev(m, std::move(d));
        *A = mh.release();
        return GrB_SUCCESS;
    });
}

// GRAPH.BULK's edge load into an EMPTY relationship tensor (src/commands/bulk_insert.rs:497 -> graph.rs:2062-2122 ->
// Tensor::set_all_from_slices, tensor.rs:333-447) as one device-side build instead of n host-side probe-and-insert steps: the
// forward UINT64 matrix (value = the pair's edge id, or MULTI_EDGE = UINT64_MAX when the pair has several edges) and the (pair key
// = src << 32 | dst, edge id) list of every edge of every multi-edge pair, sorted by (key, id) -- the entries of the reference's
// `me` store.  *multi_keys / *multi_ids are allocated with GxB_init's malloc (NULL when *nmulti == 0): the caller frees them.
GrB_Info B200_Tensor_bulk_build(GrB_Matrix *fwd, GrB_Index **multi_keys, GrB_Index **multi_ids, GrB_Index *nmulti, GrB_Index nrows,
                                GrB_Index ncols, const GrB_Index *srcs, const GrB_Index *dsts, const GrB_Index *ids, GrB_Index n) {
    CHECK_PTR(fwd); CHECK_PTR(multi_keys); CHECK_PTR(multi_ids); CHECK_PTR(nmulti);
    if (n) { CHECK_PTR(srcs); CHECK_PTR(dsts); CHECK_PTR(ids); }
    if (nrows >= ((u64)1 << 32) || ncols >= ((u64)1 << 32)) { tl_error = "bulk build: dimensions must be below 2^32"; return GrB_INVALID_VALUE; }
    return guarded([&]() {
        GpuLock g;
        std::unique_ptr<GB_Matrix_opaque> mh(new GB_Matrix_opaque());   // released to the caller only on success
        GrB_Matrix m = mh.get();
        m->type = T_UINT64; m->nrows = nrows; m->ncols = ncols;
        *multi_keys = nullptr; *multi_ids = nullptr; *nmulti = 0;
        if (n == 0) { *fwd = mh.release(); return GrB_SUCCESS; }
        ensure_init();
        DevBuf<u64> dI(n), dJ(n), dID(n), mk, mi;
        h2d(dI.ptr, (const u64 *)srcs, n);
        h2d(dJ.ptr, (const u64 *)dsts, n);
        h2d(dID.ptr, (const u64 *)ids, n);
        DevCSR out;
        bool err = false;
        u64 nm = 0;
        tensor_bulk_build(dI.ptr, dJ.ptr, dID.ptr, n, nrows, ncols, out, mk, mi, &nm, &err);
        sync_stream();
        if (err) { tl_error = "bulk build: index out of bounds"; return GrB_INDEX_OUT_OF_BOUNDS; }
        struct UserBuf {                       // handed to the caller only on success
            u64 *p = nullptr;
            ~UserBuf() { if (p) g_user_free(p); }
            u64 *release() { u64 *r = p; p = nullptr; return r; }
        } hk, hi;
        if (nm) {
            hk.p = (u64 *)g_user_malloc(nm * sizeof(u64));
            hi.p = (u64 *)g_user_malloc(nm * sizeof(u64));
            if (!hk.p || !hi.p) throw std::bad_alloc();
            d2h(hk.p, mk.ptr, nm);
            d2h(hi.p, mi.ptr, nm);
            sync_stream();
        }
        set_dev(m, std::move(out));
        *multi_keys = hk.release(); *multi_ids = hi.release(); *nmulti = nm;
        *fwd = mh.release();
        return GrB_SUCCESS;
    });
}

// ExpandInto's per-row point lookups (expand_into.rs:195-249, Tensor::get -> GrB_Matrix_extractElement) as one batched call
GrB_Info B200_Matrix_extract_pairs(GrB_Matrix A, const GrB_Index *I, const GrB_Index *J, GrB_Index n, uint8_t *found,
                                   uint64_t *values) {
    CHECK_MAT(A); CHECK_PTR(found);
    if (n) { CHECK_PTR(I); CHECK_PTR(J); }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_init();
        ensure_dev(A);
        if (n == 0) return GrB_SUCCESS;
        DevBuf<u64> dI(n), dJ(n), dV;
        DevBuf<unsigned char> dF(n);
        h2d(dI.ptr, (const u64 *)I, n);
        h2d(dJ.ptr, (const u64 *)J, n);
        if (values) dV.alloc(n);
        probe_pairs(A->dev, dI.ptr, dJ.ptr, n, dF.ptr, values ? dV.ptr : nullptr);
        d2h(found, dF.ptr, n);
        if (values) d2h(values, dV.ptr, n);
        sync_stream();
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Matrix_rmat_block(GrB_Matrix *A, int scale, uint64_t edge_factor, uint64_t seed, uint64_t lo, uint64_t hi, int by_col) {
    CHECK_PTR(A);
    return guarded([&]() {
        GpuLock g;
        ensure_init();
        std::unique_ptr<GB_Matrix_opaque> mh(new GB_Matrix_opaque());   // released to the caller only on success
        GrB_Matrix m = mh.get();
        if (scale < 1 || scale > 31 || lo > hi || hi > ((u64)1 << scale)) throw GrbError(GrB_INVALID_VALUE, "rmat_block: scale in [1, 31], 0 <= lo <= hi <= 2^scale");
        m->type = T_BOOL; m->nrows = hi - lo; m->ncols = (u64)1 << scale;
        DevCSR d;
        rmat_block_csr(scale, edge_factor, seed, lo, hi, by_col, d);
        sync_stream();
        set_dev(m, std::move(d));
        *A = mh.release();
        return GrB_SUCCESS;
    });
}


// returns every cached device block to the driver (the caching allocator otherwise keeps freed blocks for reuse)
GrB_Info B200_pool_trim(void) {
    return guarded([&]() {
        GpuLock g;
        if (ctx().ready) pool_trim();
        return GrB_SUCCESS;
    });
}
GrB_Info B200_sync(void) {
    return guarded([&]() {
        GpuLock g;   // sync_stream also delivers pending small reads: not under a submitter's feet
        if (ctx().ready) sync_stream();
        return GrB_SUCCESS;
    });
}
void *B200_stream(void) {
    try { ensure_init(); } catch (...) { return nullptr; }
    return (void *)ctx().stream;
}
uint64_t B200_get_stat(const char *name) {
    Context &c = ctx();
    std::string n = name ? name : "";
    if (n == "launches") return c.launches.load();
    if (n == "lib_launches") return c.lib_launches.load();
    if (n == "last_flops") return c.last_flops.load();
    if (n == "total_flops") return c.total_flops.load();
    if (n == "last_path") return c.last_path.load();
    if (n == "h2d_bytes") return c.h2d_bytes.load();
    if (n == "d2h_bytes") return c.d2h_bytes.load();
    if (n == "num_sms") return (uint64_t)c.num_sms;
    if (n == "l2_bytes") return (uint64_t)c.l2_bytes;
    if (n == "host_bytes") return g_host_bytes.load();     // live bytes obtained through the GxB_init allocator hooks
    if (n == "host_allocs") return g_host_allocs.load();
    return ~0ULL;
}
int B200_kernel_stats(const char *name, double *ms, uint64_t *launches, uint64_t *bytes) {
    double m[TK_COUNT_]; u64 n[TK_COUNT_], b[TK_COUNT_];
    try { timed_collect(m, n, b); } catch (...) { return -1; }
    for (int i = 0; i < TK_COUNT_; i++)
        if (name && std::string(name) == timed_name(i)) {
            if (ms) *ms = m[i];
            if (launches) *launches = n[i];
            if (bytes) *bytes = b[i];
            return 0;
        }
    return -3;
}
void B200_reset_stats(void) {
    Context &c = ctx();
    if (c.ready) { try { timed_reset(); } catch (...) {} }
    c.launches = 0; c.lib_launches = 0; c.last_flops = 0; c.total_flops = 0; c.h2d_bytes = 0; c.d2h_bytes = 0;
}
GrB_Info B200_set_option(const char *name, int64_t value) {
    Context &c = ctx();
    std::string n = name ? name : "";
    if (n == "bits_mode") c.opt_bits_mode = value;
    else if (n == "pull_mode") c.opt_pull_mode = value;
    else if (n == "small_cap") c.opt_small_cap = value;
    else if (n == "bitmap_budget") c.opt_bitmap_budget = value;
    else if (n == "bits_min_flops") c.opt_bits_min_flops = value;
    else if (n == "sync_after_op") c.opt_sync_after_op = value;
    else if (n == "hints") c.opt_hints = value;
    else if (n == "hot_pack") c.opt_hot_pack = value;
    else if (n == "hot_bytes") c.opt_hot_bytes = value;
    else if (n == "hint_streams") c.opt_hint_streams = value;
    else if (n == "hot_shuffle") c.opt_hot_shuffle = value;
    else if (n == "early_exit") c.opt_early_exit = value;
    else if (n == "pull_grid") c.opt_pull_grid = value;
    else if (n == "diag_filter") c.opt_diag_filter = value;
    else if (n == "csr_push") c.opt_csr_push = value;
    else if (n == "fused_prep") c.opt_fused_prep = value;
    else if (n == "perm_push") c.opt_perm_push = value;
    else if (n == "push_slices") c.opt_push_slices = value;
    else if (n == "union_accum") c.opt_union_accum = value;
    else if (n == "shortest_path_budget") c.opt_shortest_path_budget = value;
    // retired: the pull, the count pass and the fill have a single kernel each now, and there is no persisting-L2 window; the
    // names stay accepted so callers that set them keep working
    else if (n == "fill_kernel" || n == "fill_cap" || n == "pull_kernel" || n == "unroll" || n == "small_split" ||
             n == "count_kernel" || n == "l2_window" || n == "l2_reset") {}
    else if (n == "bfs_direction") c.opt_bfs_direction = value;
    else if (n == "bfs_sparse_exchange") c.opt_bfs_sparse_exchange = value;
    else if (n == "timing") { c.opt_timing = value; if (c.ready) timed_reset(); }
    else return GrB_INVALID_VALUE;
    return GrB_SUCCESS;
}

} // extern "C"

// ====================================================================================================================
// Serialization boundary (SURVEY 8b): GxB_Container, GxB_Vector_load / unload, GxB_Vector_serialize / deserialize.
// The reference's RDB encoder (matrix.rs:428-546, vector.rs:150-420) unloads a matrix into a container, writes the
// 608-byte struct plus the five payload vectors (x, h, p, i, b) as raw arrays, and loads it back; decode feeds
// attacker-controlled bytes through the same calls, so every length / offset below is validated before use.
// Host-side plumbing only: nothing here touches the device except fetching a device-resident matrix once.
// Layout written by unload: row-major; GxB_SPARSE (p has nrows+1 entries) when nrows < 2^32, else GxB_HYPERSPARSE
// (h = ids of the non-empty rows, p has nvec+1 entries); p, h: UINT64; i: UINT32 when ncols <= 2^32, else UINT64;
// x: one BOOL `true` (iso) for pattern matrices, UINT64[nvals] otherwise; b: empty.
// Buffers handed to the caller (unloaded arrays, blobs) come from the allocator given to GxB_init (matrix.rs:125-131),
// because the caller releases them with its own allocator (vector.rs:171-172).
// ====================================================================================================================
static size_t type_size(int code) { return code == T_BOOL ? 1 : code == T_UINT32 ? 4 : 8; }
static GrB_Type type_of(int code) { return code == T_BOOL ? GrB_BOOL : code == T_UINT32 ? GrB_UINT32 : code == T_INT64 ? GrB_INT64 : code == T_FP64 ? GrB_FP64 : GrB_UINT64; }

// replace the content of a container vector with a full (dense) array copied from `src`
static void vec_set_full(GrB_Vector v, int type, const void *src, u64 n) {
    if (v->fx) { g_user_free(v->fx); v->fx = nullptr; }
    v->idx.clear(); v->val.clear();
    v->type = type; v->n = n; v->full = true; v->fbytes = n * type_size(type);
    if (v->fbytes) {
        v->fx = g_user_malloc(v->fbytes);
        if (!v->fx) throw std::bad_alloc();
        memcpy(v->fx, src, v->fbytes);
    }
}
static void vec_set_empty(GrB_Vector v) {
    if (v->fx) { g_user_free(v->fx); v->fx = nullptr; }
    v->idx.clear(); v->val.clear();
    v->n = 0; v->full = true; v->fbytes = 0;
}
// read entry k of a full integer vector (UINT32 / UINT64 / INT64)
static bool vec_full_int(GrB_Vector v) { return v && v->full && (v->type == T_UINT32 || v->type == T_UINT64 || v->type == T_INT64); }
static u64 vec_at(GrB_Vector v, u64 k) {
    return v->type == T_UINT32 ? (u64)((const u32 *)v->fx)[k] : v->type == T_BOOL ? (u64)((const unsigned char *)v->fx)[k] : ((const u64 *)v->fx)[k];
}
static void vec_make_sparse(GrB_Vector v) {
    if (!v->full) return;
    uvec<u64> idx(v->n);
    uvec<i64> val(v->n);
    for (u64 k = 0; k < v->n; k++) { idx[k] = k; val[k] = v->fx ? (i64)vec_at(v, k) : 0; }
    if (v->fx) { g_user_free(v->fx); v->fx = nullptr; }
    v->idx = std::move(idx); v->val = std::move(val);
    v->full = false; v->fbytes = 0;
}

extern "C" {

GrB_Info GxB_Container_new(GxB_Container *Container) {
    CHECK_PTR(Container);
    return guarded([&]() {
        GxB_Container c = (GxB_Container)user_zalloc(sizeof(struct GxB_Container_struct));
        if (!c) throw std::bad_alloc();
        GrB_Vector *vs[5] = {&c->p, &c->h, &c->b, &c->i, &c->x};
        for (GrB_Vector *pv : vs) { *pv = new GB_Vector_opaque(); (*pv)->full = true; (*pv)->n = 0; }
        c->format = GxB_SPARSE; c->orientation = GrB_ROWMAJOR; c->nrows_nonempty = -1; c->ncols_nonempty = -1;
        *Container = c;
        return GrB_SUCCESS;
    });
}
GrB_Info GxB_Container_free(GxB_Container *Container) {
    if (!Container || !*Container) return GrB_SUCCESS;
    GxB_Container c = *Container;
    GrB_Vector *vs[5] = {&c->p, &c->h, &c->b, &c->i, &c->x};
    for (GrB_Vector *pv : vs) GrB_Vector_free(pv);
    if (c->Y) GrB_Matrix_free(&c->Y);
    g_user_free(c);
    *Container = nullptr;
    return GrB_SUCCESS;
}

GrB_Info GxB_unload_Matrix_into_Container(GrB_Matrix A, GxB_Container c, GrB_Descriptor) {
    CHECK_MAT(A); CHECK_PTR(c);
    if (!c->p || !c->h || !c->b || !c->i || !c->x) { tl_error = "unload: container vectors missing"; return GrB_NULL_POINTER; }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        ensure_host(A);
        const HostStore &h = A->host;
        const u64 nvec = h.hrow.size(), nnz = h.nnz();
        const bool hyper = A->nrows >= ((u64)1 << 32);
        if (hyper) {
            vec_set_full(c->p, T_UINT64, h.hptr.data(), nvec + 1);
            vec_set_full(c->h, T_UINT64, h.hrow.data(), nvec);
        } else {
            uvec<u64> p(A->nrows + 1, 0);
            for (u64 k = 0; k < nvec; k++) p[h.hrow[k] + 1] = h.hptr[k + 1] - h.hptr[k];
            for (u64 r = 0; r < A->nrows; r++) p[r + 1] += p[r];
            vec_set_full(c->p, T_UINT64, p.data(), A->nrows + 1);
            vec_set_empty(c->h);
        }
        if (A->ncols <= ((u64)1 << 32)) {
            uvec<u32> i32(nnz);
            for (u64 q = 0; q < nnz; q++) i32[q] = (u32)h.hcol[q];
            vec_set_full(c->i, T_UINT32, i32.data(), nnz);
        } else vec_set_full(c->i, T_UINT64, h.hcol.data(), nnz);
        if (A->valued()) vec_set_full(c->x, A->type, h.hval.data(), nnz);
        else { const unsigned char one = 1; vec_set_full(c->x, T_BOOL, &one, 1); }
        vec_set_empty(c->b);
        c->nrows = A->nrows; c->ncols = A->ncols; c->nvals = nnz;
        c->nrows_nonempty = (int64_t)nvec; c->ncols_nonempty = -1;
        c->format = hyper ? GxB_HYPERSPARSE : GxB_SPARSE; c->orientation = GrB_ROWMAJOR;
        c->iso = !A->valued(); c->jumbled = false;
        // the matrix keeps its handle but gives up its content and dimensions
        A->nrows = 0; A->ncols = 0;
        set_empty(A);
        return GrB_SUCCESS;
    });
}

GrB_Info GxB_load_Matrix_from_Container(GrB_Matrix A, GxB_Container c, GrB_Descriptor) {
    CHECK_MAT(A); CHECK_PTR(c);
    return guarded([&]() {
        GpuLock g;
        MultiLock lk{A};
        auto bad = [](const char *m) { throw GrbError(GrB_INVALID_OBJECT, m); };
        if (c->nrows > ((u64)1 << 60) || c->ncols > ((u64)1 << 60)) bad("load: dimensions out of range");
        if (c->orientation != GrB_ROWMAJOR) bad("load: only row-major containers are supported");
        if (c->format != GxB_SPARSE && c->format != GxB_HYPERSPARSE) bad("load: only sparse / hypersparse containers are supported");
        if (!vec_full_int(c->p) || !vec_full_int(c->i) || !c->x || !c->x->full) bad("load: p / i / x must be full vectors");
        const bool hyper = c->format == GxB_HYPERSPARSE;
        if (hyper && !vec_full_int(c->h)) bad("load: hypersparse container without h");
        const u64 nvec = hyper ? c->h->n : c->nrows;
        if (c->p->n != nvec + 1) bad("load: p has the wrong length");
        if (c->p->n && vec_at(c->p, 0) != 0) bad("load: p[0] != 0");
        const u64 nnz = c->p->n ? vec_at(c->p, nvec) : 0;
        if (nnz != c->nvals || c->i->n < nnz) bad("load: nvals / i disagree with p");
        const int xtype = c->x->type;
        if (xtype != T_BOOL && xtype != T_UINT64 && xtype != T_INT64) bad("load: unsupported value type");
        const bool iso = c->iso;
        if (c->x->n < (iso ? (nnz ? 1 : 0) : nnz)) bad("load: x too short");
        if (xtype == T_BOOL && !iso)
            for (u64 q = 0; q < nnz; q++) if (!((const unsigned char *)c->x->fx)[q]) bad("load: explicit false entries are not representable");
        if (xtype == T_BOOL && iso && nnz && !((const unsigned char *)c->x->fx)[0]) bad("load: an iso `false` pattern is not representable");
        HostStore h;
        h.clear();
        h.hcol.resize(nnz);
        if (xtype != T_BOOL) h.hval.resize(nnz);
        u64 prev_row = 0;
        for (u64 k = 0; k < nvec; k++) {
            const u64 s = vec_at(c->p, k), e = vec_at(c->p, k + 1);
            if (e < s || e > nnz) bad("load: p is not monotone");
            const u64 row = hyper ? vec_at(c->h, k) : k;
            if (row >= c->nrows || (hyper && k && row <= prev_row)) bad("load: row ids out of range or not ascending");
            prev_row = row;
            if (e == s) continue;
            for (u64 q = s; q < e; q++) {
                const u64 col = vec_at(c->i, q);
                if (col >= c->ncols) bad("load: column index out of range");
                h.hcol[q] = col;
                if (xtype != T_BOOL) h.hval[q] = iso ? ((const u64 *)c->x->fx)[0] : ((const u64 *)c->x->fx)[q];
            }
            if (c->jumbled) {   // sort the row by column, values along
                uvec<std::pair<u64, u64>> t(e - s);
                for (u64 q = s; q < e; q++) t[q - s] = {h.hcol[q], xtype != T_BOOL ? h.hval[q] : 1};
                std::sort(t.begin(), t.end());
                for (u64 q = s; q < e; q++) { h.hcol[q] = t[q - s].first; if (xtype != T_BOOL) h.hval[q] = t[q - s].second; }
            }
            for (u64 q = s + 1; q < e; q++) if (h.hcol[q] <= h.hcol[q - 1]) bad("load: duplicate or unsorted column indices");
            h.hrow.push_back(row);
            h.hptr.push_back(e);
        }
        // rows may leave gaps in p (s > previous e): compact so that hptr is contiguous
        {
            u64 w = 0;
            uvec<u64> ncol, nval;
            ncol.reserve(nnz); if (xtype != T_BOOL) nval.reserve(nnz);
            uvec<u64> nptr(1, 0);
            u64 kk = 0;
            for (u64 k = 0; k < nvec; k++) {
                const u64 s = vec_at(c->p, k), e = vec_at(c->p, k + 1);
                if (e == s) continue;
                for (u64 q = s; q < e; q++) { ncol.push_back(h.hcol[q]); if (xtype != T_BOOL) nval.push_back(h.hval[q]); }
                w += e - s; nptr.push_back(w); kk++;
            }
            h.hcol.swap(ncol); h.hval.swap(nval); h.hptr.swap(nptr);
            (void)kk;
        }
        A->type = xtype;
        A->nrows = c->nrows; A->ncols = c->ncols;
        set_empty(A);
        A->host = std::move(h);
        A->host_valid = true;
        // the container gives up its content
        vec_set_empty(c->p); vec_set_empty(c->h); vec_set_empty(c->i); vec_set_empty(c->x); vec_set_empty(c->b);
        c->nvals = 0;
        return GrB_SUCCESS;
    });
}

// V must be a full vector (the container payload vectors are); the array leaves with the caller, V becomes empty
GrB_Info GxB_Vector_unload(GrB_Vector V, void **X, GrB_Type *type, uint64_t *n, uint64_t *X_memsize, int *handling, GrB_Descriptor) {
    CHECK_PTR(V); CHECK_PTR(X); CHECK_PTR(type); CHECK_PTR(n); CHECK_PTR(X_memsize); CHECK_PTR(handling);
    return guarded([&]() {
        if (!V->full) {
            if (V->idx.size() != V->n) throw GrbError(GrB_INVALID_OBJECT, "Vector_unload: the vector is not full (every entry present)");
            // densify a sparse-API vector that happens to be full
            uvec<unsigned char> bytes(V->n * type_size(V->type));
            for (u64 k = 0; k < V->n; k++) {
                if (V->type == T_BOOL) bytes[k] = V->val[k] != 0;
                else ((u64 *)bytes.data())[k] = (u64)V->val[k];
            }
            vec_set_full(V, V->type, bytes.data(), V->n);
        }
        *X = V->fx; *type = type_of(V->type); *n = V->n; *X_memsize = V->fbytes; *handling = 0 /* GrB_DEFAULT: owned, now by the caller */;
        V->fx = nullptr; V->fbytes = 0; V->n = 0;
        return GrB_SUCCESS;
    });
}
// V adopts *X (n entries of `type`, X_memsize bytes) and *X is set to NULL
GrB_Info GxB_Vector_load(GrB_Vector V, void **X, GrB_Type type, uint64_t n, uint64_t X_memsize, int handling, GrB_Descriptor) {
    CHECK_PTR(V); CHECK_PTR(X); CHECK_PTR(type);
    return guarded([&]() {
        const int code = type->code;
        if (code != T_BOOL && code != T_UINT32 && code != T_UINT64 && code != T_INT64) throw GrbError(GrB_DOMAIN_MISMATCH, "Vector_load: unsupported type");
        if (handling != 0) throw GrbError(GrB_NOT_IMPLEMENTED, "Vector_load: read-only (GxB_IS_READONLY) arrays are not supported");
        if (n > ((u64)1 << 60) || n * type_size(code) > X_memsize) throw GrbError(GrB_INVALID_VALUE, "Vector_load: X_memsize smaller than n entries");
        if (n && !*X) throw GrbError(GrB_NULL_POINTER, "Vector_load: null array");
        if (V->fx) g_user_free(V->fx);
        V->idx.clear(); V->val.clear();
        V->type = code; V->n = n; V->full = true; V->fx = *X; V->fbytes = X_memsize;
        *X = nullptr;
        return GrB_SUCCESS;
    });
}

// ---- blob: "B2GV" | version | type | flags | n | nvals | idx[nvals] | (val[nvals] unless every value is 1) ; all little-endian u64 after the
// 16-byte head.  Opaque to the caller, like SuiteSparse's (whose blobs it does not try to read: a dump written by one
// library must be restored by the same one).
struct BlobHead { u32 magic, version; int32_t type; u32 flags; u64 n, nvals; };
static const u32 BLOB_MAGIC = 0x56473242u; // "B2GV"

GrB_Info GxB_Vector_serialize(void **blob_handle, GrB_Index *blob_size, GrB_Vector u, GrB_Descriptor) {
    CHECK_PTR(blob_handle); CHECK_PTR(blob_size); CHECK_PTR(u);
    return guarded([&]() {
        uvec<u64> idx, val;
        if (u->full) {
            idx.resize(u->n); val.resize(u->n);
            for (u64 k = 0; k < u->n; k++) { idx[k] = k; val[k] = u->type == T_BOOL ? ((const unsigned char *)u->fx)[k] : vec_at(u, k); }
        } else {
            idx = u->idx;
            val.assign(u->val.begin(), u->val.end());
        }
        bool all_one = true;
        for (u64 x : val) if (x != 1) { all_one = false; break; }
        BlobHead hd{BLOB_MAGIC, 1, u->type, all_one ? 1u : 0u, u->n, (u64)idx.size()};
        const size_t bytes = sizeof(hd) + 8 * idx.size() * (all_one ? 1 : 2);
        unsigned char *b = (unsigned char *)g_user_malloc(bytes);
        if (!b) throw std::bad_alloc();
        memcpy(b, &hd, sizeof(hd));
        memcpy(b + sizeof(hd), idx.data(), 8 * idx.size());
        if (!all_one) memcpy(b + sizeof(hd) + 8 * idx.size(), val.data(), 8 * val.size());
        *blob_handle = b; *blob_size = bytes;
        return GrB_SUCCESS;
    });
}
GrB_Info GxB_Vector_deserialize(GrB_Vector *w, GrB_Type type, const void *blob, GrB_Index blob_size, GrB_Descriptor) {
    CHECK_PTR(w); CHECK_PTR(blob);
    return guarded([&]() {
        auto bad = [](const char *m) { throw GrbError(GrB_INVALID_OBJECT, m); };
        BlobHead hd;
        if (blob_size < sizeof(hd)) bad("deserialize: blob shorter than its header");
        memcpy(&hd, blob, sizeof(hd));
        if (hd.magic != BLOB_MAGIC || hd.version != 1) bad("deserialize: not a blob written by this library");
        if (hd.type != T_BOOL && hd.type != T_UINT64 && hd.type != T_INT64 && hd.type != T_UINT32) bad("deserialize: unknown type");
        if (type && type->code != hd.type) throw GrbError(GrB_DOMAIN_MISMATCH, "deserialize: type differs from the blob's");
        const bool all_one = hd.flags & 1;
        if (hd.n > ((u64)1 << 60) || hd.nvals > hd.n || hd.nvals > (blob_size - sizeof(hd)) / (all_one ? 8 : 16)) bad("deserialize: lengths disagree with the blob size");
        if (blob_size != sizeof(hd) + 8 * hd.nvals * (all_one ? 1 : 2)) bad("deserialize: trailing or missing bytes");
        GrB_Vector v = new GB_Vector_opaque();
        v->type = hd.type; v->n = hd.n;
        v->idx.resize(hd.nvals); v->val.resize(hd.nvals);
        const unsigned char *p = (const unsigned char *)blob + sizeof(hd);
        memcpy(v->idx.data(), p, 8 * hd.nvals);
        if (all_one) std::fill(v->val.begin(), v->val.end(), 1);
        else memcpy(v->val.data(), p + 8 * hd.nvals, 8 * hd.nvals);
        for (u64 k = 0; k < hd.nvals; k++)
            if (v->idx[k] >= hd.n || (k && v->idx[k] <= v->idx[k - 1])) { delete v; bad("deserialize: indices out of range or not ascending"); }
        *w = v;
        return GrB_SUCCESS;
    });
}

GrB_Info GrB_Type_get_String(GrB_Type type, char *value, int field) {
    CHECK_PTR(type); CHECK_PTR(value);
    if (field != GrB_NAME && field != GxB_JIT_C_NAME) return GrB_INVALID_VALUE;
    const char *nm = field == GxB_JIT_C_NAME ? type->name
                   : type->code == T_BOOL ? "GrB_BOOL" : type->code == T_UINT32 ? "GrB_UINT32" : type->code == T_UINT64 ? "GrB_UINT64" : "GrB_INT64";
    strncpy(value, nm, GxB_MAX_NAME_LEN - 1);
    value[GxB_MAX_NAME_LEN - 1] = 0;
    return GrB_SUCCESS;
}
GrB_Info GxB_Type_from_name(GrB_Type *type, const char *type_name) {
    CHECK_PTR(type); CHECK_PTR(type_name);
    struct { const char *a, *b; GrB_Type t; } tab[] = {{"bool", "GrB_BOOL", GrB_BOOL}, {"uint32_t", "GrB_UINT32", GrB_UINT32},
                                                      {"uint64_t", "GrB_UINT64", GrB_UINT64}, {"int64_t", "GrB_INT64", GrB_INT64}};
    for (auto &e : tab) if (!strcmp(type_name, e.a) || !strcmp(type_name, e.b)) { *type = e.t; return GrB_SUCCESS; }
    *type = nullptr;
    tl_error = "Type_from_name: unknown type name";
    return GrB_INVALID_VALUE;
}

} // extern "C"
