// matrix.hpp -- C++ mirror of the reference's safe GraphBLAS wrapper `Matrix<T>`
// (graph/src/graph/graphblas/matrix.rs:360-1605), written against the GraphBLAS C ABI in
// include/b200grb.h exactly as the Rust file is written against bindgen's mod.rs.  The reference is
// Rust; this image has no Rust toolchain, so the host side above the C ABI is C++ (task rule 2).
// Same method names, argument meaning and error behaviour (debug-assert on GrB_Info, assert on *_new).
#pragma once
#include "../../../include/b200grb.h"
#include <atomic>
#include <cassert>
#include <cstdint>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

namespace fdb {

inline void grb_ok(GrB_Info info, const char *what) {
    if (info != GrB_SUCCESS) throw std::runtime_error(std::string(what) + " failed: " + std::to_string((int)info) + " " + B200_last_error());
}

enum class Descriptor { None, RC, RSC, RCT0, C };
inline GrB_Descriptor to_desc(Descriptor d) {
    switch (d) {
    case Descriptor::RC: return GrB_DESC_RC;
    case Descriptor::RSC: return GrB_DESC_RSC;
    case Descriptor::RCT0: return GrB_DESC_RCT0;
    case Descriptor::C: return GrB_DESC_C;
    default: return nullptr;
    }
}

// Arc<GrB_Matrix> + wait-mutex + has_pending flag (matrix.rs:360-368)
struct Handle {
    GrB_Matrix m = nullptr;
    std::mutex lock;
    std::atomic<bool> has_pending{false};
    ~Handle() { if (m) GrB_Matrix_free(&m); }
};

template <class T>
class Matrix {
    static_assert(std::is_same<T, bool>::value || std::is_same<T, uint64_t>::value, "bool or u64");
    std::shared_ptr<Handle> h;

    // pin_sparse, matrix.rs:405-426
    static void pin_sparse(GrB_Matrix m) {
        GrB_Matrix_set_INT32(m, GxB_SPARSE | GxB_HYPERSPARSE, GxB_SPARSITY_CONTROL);
        GrB_Matrix_set_INT32(m, GrB_ROWMAJOR, GrB_STORAGE_ORIENTATION_HINT);
    }

  public:
    using Item = typename std::conditional<std::is_same<T, bool>::value, std::tuple<uint64_t, uint64_t>,
                                           std::tuple<uint64_t, uint64_t, uint64_t>>::type;
    Matrix() {}
    Matrix(uint64_t nrows, uint64_t ncols) { // matrix.rs:1119 / :1214
        h = std::make_shared<Handle>();
        grb_ok(GrB_Matrix_new(&h->m, std::is_same<T, bool>::value ? GrB_BOOL : GrB_UINT64, nrows, ncols), "GrB_Matrix_new");
        pin_sparse(h->m);
    }
    static Matrix adopt(GrB_Matrix raw, bool pending) {
        Matrix r;
        r.h = std::make_shared<Handle>();
        r.h->m = raw;
        r.h->has_pending = pending;
        return r;
    }
    bool valid() const { return (bool)h; }
    GrB_Matrix inner() const { return h->m; }                 // matrix.rs:720
    bool is_shared() const { return h.use_count() > 1; }

    Matrix &into_hyper() {                                    // matrix.rs:558-575
        GrB_Matrix_set_INT32(h->m, GxB_HYPERSPARSE, GxB_SPARSITY_CONTROL);
        GrB_Matrix_set_INT32(h->m, 0, GxB_HYPER_HASH);
        return *this;
    }
    // matrix.rs:596-625: number of stored vectors of a hypersparse matrix, -1 otherwise
    int64_t hyper_vector_count() const {
        int32_t st = 0;
        GrB_Matrix_get_INT32(h->m, &st, GxB_SPARSITY_STATUS);
        if (st != GxB_HYPERSPARSE) return -1;
        GxB_Iterator it = nullptr;
        grb_ok(GxB_Iterator_new(&it), "Iterator_new");
        grb_ok(GxB_rowIterator_attach(it, h->m, nullptr), "attach");
        int64_t k = (int64_t)GxB_rowIterator_kount(it);
        GxB_Iterator_free(&it);
        return k;
    }
    uint64_t nrows() const { GrB_Index n = 0; grb_ok(GrB_Matrix_nrows(&n, h->m), "nrows"); return n; }
    uint64_t ncols() const { GrB_Index n = 0; grb_ok(GrB_Matrix_ncols(&n, h->m), "ncols"); return n; }
    uint64_t nvals() const { GrB_Index n = 0; grb_ok(GrB_Matrix_nvals(&n, h->m), "nvals"); return n; }
    bool pending() const { int32_t v = 0; grb_ok(GrB_Matrix_get_INT32(h->m, &v, GxB_WILL_WAIT), "get WILL_WAIT"); return v == 1; }
    bool is_synced() const { return !h->has_pending.load(std::memory_order_relaxed); }
    void mark_pending() { h->has_pending.store(true, std::memory_order_relaxed); }

    void wait() const {                                       // matrix.rs:781-796
        if (!h->has_pending.load(std::memory_order_acquire)) return;
        std::lock_guard<std::mutex> g(h->lock);
        if (!h->has_pending.load(std::memory_order_relaxed)) return;
        grb_ok(GrB_Matrix_wait(h->m, GrB_MATERIALIZE), "GrB_Matrix_wait");
        h->has_pending.store(false, std::memory_order_release);
    }
    void clear() { grb_ok(GrB_Matrix_clear(h->m), "clear"); h->has_pending = false; }
    void resize(uint64_t r, uint64_t c) { grb_ok(GrB_Matrix_resize(h->m, r, c), "resize"); mark_pending(); }

    Matrix dup() const {                                      // matrix.rs:1062-1114
        bool pend = h->has_pending.load(std::memory_order_acquire);
        std::unique_lock<std::mutex> g;
        if (pend) g = std::unique_lock<std::mutex>(h->lock);
        bool dup_pending = pend ? h->has_pending.load(std::memory_order_relaxed) : false;
        GrB_Matrix out = nullptr;
        grb_ok(GrB_Matrix_dup(&out, h->m), "GrB_Matrix_dup");
        int32_t hh = 1;
        GrB_Matrix_get_INT32(h->m, &hh, GxB_HYPER_HASH);
        if (hh == 0) GrB_Matrix_set_INT32(out, 0, GxB_HYPER_HASH);
        return adopt(out, dup_pending);
    }
    Matrix grown(uint64_t nr, uint64_t nc) const {            // matrix.rs:700-715
        uint64_t r0 = nrows(), c0 = ncols();
        if (!(nr >= r0 && nc >= c0)) throw std::logic_error("grown must not shrink");
        Matrix out = dup();
        if (nr != r0 || nc != c0) out.resize(nr, nc);
        return out;
    }
    Matrix transpose() const {                                // matrix.rs:633-662
        Matrix t(ncols(), nrows());
        t.h->has_pending = true;
        grb_ok(GrB_transpose(t.h->m, nullptr, nullptr, h->m, nullptr), "GrB_transpose");
        return t;
    }

    // ---- element access ----
    void set(uint64_t i, uint64_t j, T v) {                   // matrix.rs:1143 / :1264
        if (std::is_same<T, bool>::value) grb_ok(GrB_Matrix_setElement_BOOL(h->m, (bool)v, i, j), "setElement");
        else grb_ok(GrB_Matrix_setElement_UINT64(h->m, (uint64_t)v, i, j), "setElement");
        mark_pending();
    }
    bool get(uint64_t i, uint64_t j, T *out = nullptr) const { // matrix.rs:1158 / :1248 (None => false)
        GrB_Info info;
        if (std::is_same<T, bool>::value) { bool b = false; info = GrB_Matrix_extractElement_BOOL(&b, h->m, i, j); if (out) *out = (T)b; }
        else { uint64_t u = 0; info = GrB_Matrix_extractElement_UINT64(&u, h->m, i, j); if (out) *out = (T)u; }
        return info == GrB_SUCCESS;
    }
    bool contains(uint64_t i, uint64_t j) const { return GxB_Matrix_isStoredElement(h->m, i, j) == GrB_SUCCESS; }
    void remove(uint64_t i, uint64_t j) { grb_ok(GrB_Matrix_removeElement(h->m, i, j), "removeElement"); mark_pending(); }

    void build(const std::vector<uint64_t> &rows, const std::vector<uint64_t> &cols, const std::vector<uint64_t> *vals = nullptr) {
        assert(rows.size() == cols.size());                   // matrix.rs:1186-1210 / :1281-1303
        if (rows.empty()) return;
        if (std::is_same<T, bool>::value) {
            GrB_Scalar s = nullptr;
            grb_ok(GrB_Scalar_new(&s, GrB_BOOL), "Scalar_new");
            grb_ok(GrB_Scalar_setElement_BOOL(s, true), "Scalar_set");
            GrB_Info info = GxB_Matrix_build_Scalar(h->m, rows.data(), cols.data(), s, rows.size());
            GrB_Scalar_free(&s);
            grb_ok(info, "GxB_Matrix_build_Scalar");
        } else {
            assert(vals && vals->size() == rows.size());
            grb_ok(GrB_Matrix_build_UINT64(h->m, rows.data(), cols.data(), vals->data(), rows.size(), GxB_ANY_UINT64), "build_UINT64");
        }
        mark_pending();
    }

    // ---- bulk algebra ----
    template <class TB> void lmxm(const Matrix<TB> &b) {       // matrix.rs:930-947
        grb_ok(GrB_mxm(h->m, nullptr, nullptr, GxB_ANY_PAIR_BOOL, h->m, b.inner(), nullptr), "GrB_mxm");
        mark_pending();
    }
    template <class TB> void rmxm(const Matrix<TB> &b) {       // matrix.rs:951-968
        grb_ok(GrB_mxm(h->m, nullptr, nullptr, GxB_ANY_PAIR_BOOL, b.inner(), h->m, nullptr), "GrB_mxm");
        mark_pending();
    }
    template <class TB> uint64_t intersection_nvals(const Matrix<TB> &b) const { // matrix.rs:743-761
        Matrix<bool> t(nrows(), ncols());
        grb_ok(GrB_Matrix_eWiseMult_Semiring(t.inner(), nullptr, nullptr, GxB_ANY_PAIR_BOOL, h->m, b.inner(), nullptr), "eWiseMult");
        return t.nvals();
    }
    template <class U> void remove_all(const Matrix<U> &b) {   // matrix.rs:824-833
        grb_ok(GrB_transpose(h->m, b.inner(), nullptr, h->m, GrB_DESC_RCT0), "GrB_transpose RCT0");
        mark_pending();
    }
    void select(const Matrix<bool> &mask, const Matrix &a) {   // matrix.rs:835-845
        grb_ok(GrB_transpose(h->m, mask.inner(), nullptr, a.inner(), GrB_DESC_RCT0), "GrB_transpose RCT0");
        mark_pending();
    }
    // self<mask> = a (+) b ; (+) = ANY for bool, SECOND for u64 (matrix.rs:257-281, 852-874)
    template <class TB>
    void element_wise_add(const Matrix<bool> *mask, const Matrix *a, const Matrix<TB> *b, Descriptor d = Descriptor::None) {
        GrB_BinaryOp op = std::is_same<T, bool>::value ? GxB_ANY_BOOL : GrB_SECOND_UINT64;
        grb_ok(GrB_Matrix_eWiseAdd_BinaryOp(h->m, mask ? mask->inner() : nullptr, nullptr, op, a ? a->inner() : h->m,
                                            b ? b->inner() : h->m, to_desc(d)), "eWiseAdd");
        mark_pending();
    }
    template <class TB>
    void element_wise_multiply(const Matrix<bool> *mask, const Matrix<bool> *a, const Matrix<TB> *b, Descriptor d = Descriptor::None) {
        grb_ok(GrB_Matrix_eWiseMult_Semiring(h->m, mask ? mask->inner() : nullptr, nullptr, GxB_ANY_PAIR_BOOL,
                                             a ? a->inner() : h->m, b ? b->inner() : h->m, to_desc(d)), "eWiseMult");
        mark_pending();
    }
    template <class TB> void set_pattern(const Matrix<bool> *mask, const Matrix<TB> &a, Descriptor d = Descriptor::None) {
        grb_ok(GrB_Matrix_apply(h->m, mask ? mask->inner() : nullptr, GxB_ANY_BOOL, GxB_ONE_BOOL, a.inner(), to_desc(d)), "apply");
        mark_pending();                                        // matrix.rs:906-924
    }

    // Matrix::<bool>::delta_lmxm, matrix.rs:1317-1402, statement for statement
    template <class TV>
    void delta_lmxm(const Matrix<TV> &m, const Matrix<TV> &dp, const Matrix<bool> &dm) {
        static_assert(std::is_same<T, bool>::value, "delta_lmxm is defined on Matrix<bool>");
        dp.wait();
        dm.wait();
        uint64_t dp_nvals = dp.nvals(), dm_nvals = dm.nvals();
        if (dp_nvals == 0 && dm_nvals == 0) { lmxm(m); return; }
        uint64_t nr = nrows(), nc = m.ncols();
        Matrix<bool> mask, accum;
        if (dm_nvals > 0) {
            Matrix<bool> mk(nr, nc);
            grb_ok(GrB_mxm(mk.inner(), nullptr, nullptr, GxB_ANY_PAIR_BOOL, h->m, dm.inner(), nullptr), "GrB_mxm mk");
            if (mk.nvals() > 0) mask = mk;
        }
        if (dp_nvals > 0) {
            Matrix<bool> ac(nr, nc);
            grb_ok(GrB_mxm(ac.inner(), nullptr, nullptr, GxB_ANY_PAIR_BOOL, h->m, dp.inner(), nullptr), "GrB_mxm ac");
            if (ac.nvals() > 0) accum = ac;
        }
        grb_ok(GrB_mxm(h->m, mask.valid() ? mask.inner() : nullptr, nullptr, GxB_ANY_PAIR_BOOL, h->m, m.inner(),
                       mask.valid() ? GrB_DESC_RSC : nullptr), "GrB_mxm main");
        if (accum.valid()) element_wise_add<bool>(nullptr, nullptr, &accum);
        mark_pending();
    }
    // the same product as one library call (B200_Matrix_delta_lmxm): same result and flops, the delta terms applied in place
    template <class TV>
    void delta_lmxm_fused(const Matrix<TV> &m, const Matrix<TV> &dp, const Matrix<bool> &dm) {
        static_assert(std::is_same<T, bool>::value, "delta_lmxm is defined on Matrix<bool>");
        dp.wait();
        dm.wait();
        grb_ok(B200_Matrix_delta_lmxm(h->m, m.inner(), dp.inner(), dm.inner()), "B200_Matrix_delta_lmxm");
        mark_pending();
    }
    // the union hop over several relationship types as one library call (B200_Matrix_union_lmxm):
    // self <- self * U_t (m[t] \ dm[t]) u dp[t], exact; the deltas' pending tuples must be finished by the caller
    void union_lmxm(const std::vector<GrB_Matrix> &m, const std::vector<GrB_Matrix> &dp, const std::vector<GrB_Matrix> &dm) {
        static_assert(std::is_same<T, bool>::value, "union_lmxm is defined on Matrix<bool>");
        grb_ok(B200_Matrix_union_lmxm(h->m, m.data(), dp.data(), dm.data(), (int)m.size()), "B200_Matrix_union_lmxm");
        mark_pending();
    }

    // ---- iteration: the reference's loop over the C row iterator (matrix.rs:1471-1605) ----
    class Iter {
        std::shared_ptr<Handle> keep;
        GxB_Iterator it = nullptr;
        bool depleted = true;
        uint64_t max_row = 0;
        void skip_empty(GrB_Info info) {
            while (info == GrB_NO_VALUE && GxB_rowIterator_getRowIndex(it) < max_row) info = GxB_rowIterator_nextRow(it);
            depleted = info != GrB_SUCCESS || GxB_rowIterator_getRowIndex(it) > max_row;
        }
      public:
        Iter() {}
        Iter(const Matrix &m, uint64_t min_row, uint64_t max_row_) : keep(m.h), max_row(max_row_) {
            grb_ok(GxB_Iterator_new(&it), "Iterator_new");
            grb_ok(GxB_rowIterator_attach(it, m.h->m, nullptr), "rowIterator_attach");
            skip_empty(GxB_rowIterator_seekRow(it, min_row));
        }
        Iter(Iter &&o) noexcept : keep(std::move(o.keep)), it(o.it), depleted(o.depleted), max_row(o.max_row) { o.it = nullptr; }
        Iter &operator=(Iter &&o) noexcept {
            if (this != &o) { if (it) GxB_Iterator_free(&it); keep = std::move(o.keep); it = o.it; depleted = o.depleted; max_row = o.max_row; o.it = nullptr; }
            return *this;
        }
        Iter(const Iter &) = delete;
        Iter &operator=(const Iter &) = delete;
        ~Iter() { if (it) GxB_Iterator_free(&it); }
        void seek(uint64_t min_row, uint64_t max_row_) { max_row = max_row_; skip_empty(GxB_rowIterator_seekRow(it, min_row)); }
        bool next(Item &out) {
            if (depleted || !it) return false;
            uint64_t r = GxB_rowIterator_getRowIndex(it), c = GxB_rowIterator_getColIndex(it);
            assign(out, r, c, GxB_Iterator_get_UINT64(it));
            if (GxB_rowIterator_nextCol(it) != GrB_SUCCESS) skip_empty(GxB_rowIterator_nextRow(it));
            return true;
        }
      private:
        static void assign(std::tuple<uint64_t, uint64_t> &o, uint64_t r, uint64_t c, uint64_t) { o = std::make_tuple(r, c); }
        static void assign(std::tuple<uint64_t, uint64_t, uint64_t> &o, uint64_t r, uint64_t c, uint64_t v) { o = std::make_tuple(r, c, v); }
    };
    Iter iter(uint64_t min_row = 0, uint64_t max_row = UINT64_MAX) const { return Iter(*this, min_row, max_row); }
};

} // namespace fdb
