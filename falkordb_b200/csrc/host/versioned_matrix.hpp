// versioned_matrix.hpp -- C++ mirror of the reference's delta matrix `VersionedMatrix<bool>`
// (graph/src/graph/graphblas/versioned_matrix.rs:1-1253): base `m` + pending adds `dp` + tombstones `dm`,
// effective state (m \ dm) U dp, copy-on-write layers (graph/src/graph/cow.rs:43-91), the sqrt fold policy
// (:140-200) and the fold itself (flush :892-938) -- the eWiseAdd / masked-copy half of the hot path.
// Written against the same C ABI calls the Rust file makes; every GraphBLAS bulk call lands in libb200grb.so.
#pragma once
#include "matrix.hpp"
#include "serial.hpp"
#include <algorithm>
#include <optional>

namespace fdb {

// ---- fold policy, versioned_matrix.rs:140-200 ----
static const uint64_t WRITE_FOLD_K = 20500000ULL;
static const uint64_t READ_FOLD_K = 82000ULL;
static const uint64_t MIN_FOLD_DELTA = 256ULL;

inline uint64_t sat_mul(uint64_t a, uint64_t b) {
    unsigned __int128 p = (unsigned __int128)a * b;
    return p > (unsigned __int128)UINT64_MAX ? UINT64_MAX : (uint64_t)p;
}
inline bool fold_balance(uint64_t delta_nvals, uint64_t tx_added, uint64_t base_nvals, uint64_t k) {
    return tx_added > 0 && delta_nvals >= MIN_FOLD_DELTA &&
           (sat_mul(delta_nvals, 2) >= base_nvals || sat_mul(delta_nvals, delta_nvals) >= sat_mul(k, tx_added));
}
inline bool should_fold(uint64_t d, uint64_t tx, uint64_t base) { return fold_balance(d, tx, base, WRITE_FOLD_K); }
inline bool should_fold_read(uint64_t d, uint64_t tx, uint64_t base) { return fold_balance(d, tx, base, READ_FOLD_K); }
inline bool delta_dominates_base(uint64_t d, uint64_t base) { return d >= MIN_FOLD_DELTA && sat_mul(d, 2) >= base; }

// ---- Cow, cow.rs:43-91 ----
template <class M>
class Cow {
    M inner;
    bool dup_ = false;
  public:
    Cow() {}
    explicit Cow(M m) : inner(std::move(m)) {}
    Cow new_version() const { Cow c; c.inner = inner; c.dup_ = true; return c; }
    void replace(M m) { inner = std::move(m); dup_ = false; }
    const M &get() const { return inner; }
    M &get_mut() { if (dup_) { inner = inner.dup(); dup_ = false; } return inner; }
};

// ---- Delta<T>, versioned_matrix.rs:214-469 ----
template <class T>
class Delta {
    Cow<Matrix<T>> layer;
    mutable std::atomic<uint64_t> count{0};
    uint64_t tx_nvals = 0;
    mutable std::atomic<bool> fold{false};
  public:
    Delta() {}
    explicit Delta(Matrix<T> l) { uint64_t c = l.nvals(); l.into_hyper(); layer = Cow<Matrix<T>>(l); count = c; }
    Delta(const Delta &o) : layer(o.layer), count(o.count.load()), tx_nvals(o.tx_nvals), fold(o.fold.load()) {}
    Delta &operator=(const Delta &o) { layer = o.layer; count = o.count.load(); tx_nvals = o.tx_nvals; fold = o.fold.load(); return *this; }

    const Matrix<T> &m() const { return layer.get(); }
    Delta transposed() const { Delta d(*this); Matrix<T> t = layer.get().transpose(); t.into_hyper(); d.layer = Cow<Matrix<T>>(t); return d; }
    Delta new_version(bool f) const {
        Delta d;
        uint64_t c = get_count();
        d.layer = layer.new_version(); d.count = c; d.tx_nvals = c; d.fold = f;
        return d;
    }
    uint64_t get_count() const { return count.load(std::memory_order_relaxed); }
    void resync() const { layer.get().wait(); count.store(layer.get().nvals(), std::memory_order_relaxed); }
    void latch(bool decision) const { if (decision) fold.store(true, std::memory_order_relaxed); }
    bool fold_decision(bool (*policy)(uint64_t, uint64_t, uint64_t), uint64_t base) const {
        uint64_t c = get_count();
        return fold.load(std::memory_order_relaxed) || policy(c, c > tx_nvals ? c - tx_nvals : 0, base);
    }
    bool folding() const { return fold.load(std::memory_order_relaxed); }
    bool take_fold() { return fold.exchange(false, std::memory_order_relaxed) && layer.get().nvals() > 0; }
    void clear(uint64_t nrows, uint64_t ncols) {
        Matrix<T> e(nrows, ncols);
        e.into_hyper();
        layer.replace(e);
        count = 0; tx_nvals = 0; fold = false;
    }
    void replace(Matrix<T> l) { l.into_hyper(); layer.replace(l); }
    void resize(uint64_t r, uint64_t c) { layer_mut().resize(r, c); }
    Matrix<T> &layer_mut() { return layer.get_mut(); }
    void erase(uint64_t i, uint64_t j) { layer_mut().remove(i, j); uint64_t c = count.load(); count = c ? c - 1 : 0; }
    void insert(uint64_t i, uint64_t j, T v = (T)1) { layer_mut().set(i, j, v); count++; }   // :416-423 / :460-468
    // self<mask> = mask n base  (versioned_matrix.rs:428-436)
    template <class TV> void tombstone_masked(const Matrix<bool> &mask, const Matrix<TV> &base) {
        static_assert(std::is_same<T, bool>::value, "tombstones are a bool layer");
        layer_mut().template element_wise_multiply<TV>(&mask, &mask, &base);
        resync();
    }
    void remove_all(const Matrix<bool> &mask) { layer_mut().remove_all(mask); resync(); }
};
typedef Delta<bool> DeltaBool;

// ---- effective-content iterator over three layers, versioned_matrix.rs:1116-1253 (`Iter::from_layers`) ----
template <class T>
class LayerIter {
  public:
    typedef typename Matrix<T>::Item Item;
  private:
    typedef std::tuple<uint64_t, uint64_t> Pos;
    typename Matrix<T>::Iter mit, dpit;
    Matrix<bool>::Iter dmit;
    bool has_dp = false, has_dm = false;
    std::optional<Item> m_next, dp_next;
    std::optional<Pos> dm_next;
    static Pos pos(const std::tuple<uint64_t, uint64_t> &t) { return t; }
    static Pos pos(const std::tuple<uint64_t, uint64_t, uint64_t> &t) { return Pos(std::get<0>(t), std::get<1>(t)); }
  public:
    LayerIter(const Matrix<T> &m, const Matrix<T> &dp, const Matrix<bool> &dm, uint64_t min_row, uint64_t max_row) {
        mit = m.iter(min_row, max_row);
        if (dm.nvals() != 0) { dmit = dm.iter(min_row, max_row); has_dm = true; Pos t; if (dmit.next(t)) dm_next = t; }
        if (dp.nvals() != 0) { dpit = dp.iter(min_row, max_row); has_dp = true; }
    }
    void seek(uint64_t min_row, uint64_t max_row) {
        mit.seek(min_row, max_row);
        m_next.reset();
        if (has_dp) dpit.seek(min_row, max_row);
        dp_next.reset();
        if (has_dm) { dmit.seek(min_row, max_row); dm_next.reset(); Pos t; if (dmit.next(t)) dm_next = t; }
    }
    bool next(Item &out) {
        Item t;
        Pos d;
        if (!m_next && mit.next(t)) m_next = t;
        while (m_next) {
            Pos mp = pos(*m_next);
            while (dm_next && *dm_next < mp) { dm_next.reset(); if (has_dm && dmit.next(d)) dm_next = d; }
            if (dm_next && *dm_next == mp) {
                dm_next.reset();
                if (has_dm && dmit.next(d)) dm_next = d;
                m_next.reset();
                if (mit.next(t)) m_next = t;
            } else break;
        }
        if (!dp_next && has_dp && dpit.next(t)) dp_next = t;
        if (m_next && dp_next) {
            Pos mp = pos(*m_next), dpp = pos(*dp_next);
            if (dpp <= mp) {
                if (dpp == mp) m_next.reset();   // shadowed: dp yields the live value
                out = *dp_next; dp_next.reset();
            } else { out = *m_next; m_next.reset(); }
            return true;
        }
        if (m_next) { out = *m_next; m_next.reset(); return true; }
        if (dp_next) { out = *dp_next; dp_next.reset(); return true; }
        return false;
    }
};

// ---- VersionedMatrix<bool>, versioned_matrix.rs:480-1080 ----
class VersionedMatrix {
    Cow<Matrix<bool>> m_;
    DeltaBool dp_, dm_;
    mutable std::atomic<bool> needs_flush{false};

  public:
    VersionedMatrix() {}
    VersionedMatrix(uint64_t nrows, uint64_t ncols)
        : m_(Matrix<bool>(nrows, ncols)), dp_(Matrix<bool>(nrows, ncols)), dm_(Matrix<bool>(nrows, ncols)) {}
    VersionedMatrix(const VersionedMatrix &o) : m_(o.m_), dp_(o.dp_), dm_(o.dm_), needs_flush(o.needs_flush.load()) {}
    VersionedMatrix &operator=(const VersionedMatrix &o) { m_ = o.m_; dp_ = o.dp_; dm_ = o.dm_; needs_flush = o.needs_flush.load(); return *this; }
    static VersionedMatrix from_matrix(Matrix<bool> m) {       // :877-890
        m.wait();
        VersionedMatrix v;
        uint64_t r = m.nrows(), c = m.ncols();
        v.m_ = Cow<Matrix<bool>>(m);
        v.dp_ = DeltaBool(Matrix<bool>(r, c));
        v.dm_ = DeltaBool(Matrix<bool>(r, c));
        return v;
    }

    const Matrix<bool> &m() const { return m_.get(); }
    const Matrix<bool> &dp() const { return dp_.m(); }
    const Matrix<bool> &dm() const { return dm_.m(); }
    uint64_t nrows() const { return m().nrows(); }
    uint64_t ncols() const { return m().ncols(); }

    void wait() const {                                        // :545-569
        if (dp().is_synced() && dm().is_synced()) return;
        dp_.resync();
        dm_.resync();
        uint64_t base = m().nvals();
        dp_.latch(dp_.fold_decision(should_fold_read, base));
        dm_.latch(dm_.fold_decision(should_fold_read, base));
    }
    void wait_base() const { m().wait(); }
    void wait_all() const { m().wait(); dp().wait(); dm().wait(); }
    bool is_synced() const { return m().is_synced() && dp().is_synced() && dm().is_synced(); }

    Matrix<bool> extract() const {                             // :609-620
        wait();
        Matrix<bool> out(nrows(), ncols());
        out.set_pattern<bool>(nullptr, m());
        if (dm().nvals() > 0) out.remove_all(dm());
        if (dp().nvals() > 0) out.set_pattern<bool>(nullptr, dp());
        return out;
    }
    uint64_t nvals() const { wait(); return m().nvals() + dp().nvals() - dm().nvals(); }   // :629-632

    bool get(uint64_t i, uint64_t j) const {                    // :819-835
        wait();
        if (m().get(i, j)) return !dm().get(i, j);
        return dp().get(i, j);
    }
    void set(uint64_t i, uint64_t j) {                          // :844-857
        flush();
        if (m().get(i, j)) dm_.erase(i, j);
        else dp_.insert(i, j);
    }
    void remove(uint64_t i, uint64_t j) {                       // :780-791
        flush();
        if (m().get(i, j)) dm_.insert(i, j);
        else dp_.erase(i, j);
    }
    // set / remove with the base probe m().get(i, j) supplied by the caller (a write plan read it on the device): the same Delta
    // calls, no read of m
    void set_known(uint64_t i, uint64_t j, bool in_base) {
        flush();
        if (in_base) dm_.erase(i, j);
        else dp_.insert(i, j);
    }
    void remove_known(uint64_t i, uint64_t j, bool in_base) {
        flush();
        if (in_base) dm_.insert(i, j);
        else dp_.erase(i, j);
    }
    void remove_mask(const Matrix<bool> &mask) {                // :799-816
        flush();
        m().wait();
        dm_.tombstone_masked(mask, m());
        dp_.remove_all(mask);
    }
    template <bool NEW>
    void set_all(const std::vector<std::pair<uint64_t, uint64_t>> &entries) {  // :1006-1035
        flush();
        dm().wait();
        if (dm().nvals() == 0) {
            for (auto &e : entries) {
                if (!NEW && m().get(e.first, e.second)) continue;
                dp_.insert(e.first, e.second);
            }
        } else {
            for (auto &e : entries) set(e.first, e.second);
        }
    }

    // set_all with its per-entry m.get as one B200_Matrix_extract_pairs call (made only when a probe is read): the same Delta calls
    template <bool NEW>
    void set_all_dev(const std::vector<std::pair<uint64_t, uint64_t>> &entries) {
        flush();
        dm().wait();
        const bool dm_empty = dm().nvals() == 0;
        std::vector<uint8_t> in_base(entries.size(), 0);
        if (!entries.empty() && (!NEW || !dm_empty)) {
            std::vector<uint64_t> I(entries.size()), J(entries.size());
            for (size_t k = 0; k < entries.size(); k++) { I[k] = entries[k].first; J[k] = entries[k].second; }
            grb_ok(B200_Matrix_extract_pairs(m().inner(), I.data(), J.data(), I.size(), in_base.data(), nullptr),
                   "B200_Matrix_extract_pairs");
        }
        if (dm_empty) {
            for (size_t k = 0; k < entries.size(); k++) {
                if (!NEW && in_base[k]) continue;
                dp_.insert(entries[k].first, entries[k].second);
            }
        } else {
            for (size_t k = 0; k < entries.size(); k++) set_known(entries[k].first, entries[k].second, in_base[k] != 0);
        }
    }
    // the two Delta counters (dp, dm)
    void counts(uint64_t *out2) const { out2[0] = dp_.get_count(); out2[1] = dm_.get_count(); }

    void flush() {                                              // :892-938
        if (!needs_flush.load(std::memory_order_relaxed)) return;
        wait_all();
        bool fold_dp = dp_.take_fold();
        bool fold_dm = dm_.take_fold();
        if (fold_dp || fold_dm) {
            uint64_t nr = nrows(), nc = ncols();
            Matrix<bool> new_m(nr, nc);
            if (fold_dp && fold_dm) new_m.element_wise_add<bool>(&dm(), &m(), &dp(), Descriptor::RC); // new_m<!dm,replace> = m U dp
            else if (fold_dp) new_m.element_wise_add<bool>(nullptr, &m(), &dp());
            else new_m.select(dm(), m());                                                           // new_m<!dm,replace> = m
            new_m.wait();
            m_.replace(new_m);
            if (fold_dp) dp_.clear(nr, nc);
            if (fold_dm) dm_.clear(nr, nc);
        }
        needs_flush.store(false, std::memory_order_relaxed);
    }
    void fold_latched() {                                       // :948-954
        wait();
        if (dp_.folding() || dm_.folding()) { needs_flush = true; flush(); }
    }
    bool is_empty_fast() const { return m().nvals() == 0 && dp_.get_count() == 0; }
    void fold_oversized() {                                     // :972-986
        uint64_t base = m().nvals();
        bool odp = delta_dominates_base(dp_.get_count(), base), odm = delta_dominates_base(dm_.get_count(), base);
        if (odp || odm) {
            dp_.latch(odp);
            dm_.latch(odm);
            needs_flush = true;
            flush();
        }
    }
    VersionedMatrix dup() const {                               // :1051-1061
        uint64_t base = m().nvals();
        bool fdp = dp_.fold_decision(should_fold, base), fdm = dm_.fold_decision(should_fold, base);
        VersionedMatrix v;
        v.m_ = m_.new_version();
        v.dp_ = dp_.new_version(fdp);
        v.dm_ = dm_.new_version(fdm);
        v.needs_flush = fdp || fdm;
        return v;
    }
    VersionedMatrix transpose() const {                         // :1070-1079
        VersionedMatrix v;
        v.m_ = Cow<Matrix<bool>>(m().transpose());
        v.dp_ = dp_.transposed();
        v.dm_ = dm_.transposed();
        v.needs_flush = needs_flush.load();
        return v;
    }
    void resize(uint64_t nr, uint64_t nc) {                     // :656-756 (grow = fold everything into a fresh base)
        if (nr < nrows() || nc < ncols()) {
            flush();
            m_.get_mut().resize(nr, nc);
            dp_.resize(nr, nc);
            dm_.resize(nr, nc);
            return;
        }
        wait_all();
        if (dp().nvals() == 0 && dm().nvals() == 0) {
            Matrix<bool> g = m().grown(nr, nc);
            g.wait();
            m_.replace(g);
        } else {
            // (m \ dm) U dp at the new dims.  The reference streams a 3-way iterator merge into build();
            // here the same set expression runs as two bulk calls on the device.
            Matrix<bool> merged = extract();
            Matrix<bool> g = merged.grown(nr, nc);
            g.wait();
            m_.replace(g);
        }
        dp_.clear(nr, nc);
        dm_.clear(nr, nc);
        needs_flush = false;
    }

    // <VersionedMatrix<V> as Encode<19> / Decode<19>>, versioned_matrix.rs:1082-1113: the three layers in order; decoded deltas
    // have no owning transaction (tx_nvals = 0), so the write fold policy sees the whole delta as freshly added
    void encode(Stream &w) const {
        encode_matrix(m(), w);
        encode_matrix(dp(), w);
        encode_matrix(dm(), w);
    }
    static VersionedMatrix decode(Stream &r) {
        Matrix<bool> m = decode_matrix<bool>(r), dp = decode_matrix<bool>(r), dm = decode_matrix<bool>(r);
        uint64_t base = m.nvals();
        VersionedMatrix v;
        v.m_ = Cow<Matrix<bool>>(m);
        v.dp_ = DeltaBool(dp);
        v.dm_ = DeltaBool(dm);
        v.dp_.latch(v.dp_.fold_decision(should_fold, base));
        v.dm_.latch(v.dm_.fold_decision(should_fold, base));
        v.needs_flush = v.dp_.folding() || v.dm_.folding();
        return v;
    }

    typedef LayerIter<bool> Iter;   // sorted 3-way merge (m \ dm) U dp
    Iter iter(uint64_t min_row = 0, uint64_t max_row = UINT64_MAX) const { wait(); return Iter(m(), dp(), dm(), min_row, max_row); }
};

} // namespace fdb
