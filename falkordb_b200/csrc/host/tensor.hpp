// tensor.hpp -- C++ mirror of the reference's per-relationship-type edge store `Tensor`
// (graph/src/graph/graphblas/tensor.rs:184-1047): forward adjacency as three UINT64 delta layers whose values are
// inline edge ids (`m`, `dp`, `dm`), a bool backward adjacency `mt`, and the lazy multi-edge id store `me`
// (2^60 x 2^60, keyed by (src<<32)|dst).  It is the operand provider of the hot path: CondTraverse multiplies by
// fwd_m()/fwd_dp()/fwd_dm() through Matrix<bool>::delta_lmxm (cond_traverse.rs:83), and the ANY_PAIR kernels never
// read the u64 values -- which is why edge id 0 must survive every structural round trip (tensor.rs:1427-1476).
#pragma once
#include "versioned_matrix.hpp"
#include <algorithm>
#include <map>
#include <unordered_map>

namespace fdb {

static const uint64_t GrB_INDEX_MAX_ = ((uint64_t)1 << 60) - 1; // tensor.rs:142
static const uint64_t MULTI_EDGE = UINT64_MAX;                  // tensor.rs:206

inline uint64_t compound_key(uint64_t src, uint64_t dst) {      // tensor.rs:154-163
    if (src > 0xFFFFFFFFULL || dst > 0xFFFFFFFFULL) throw std::logic_error("Tensor compound key overflow");
    return (src << 32) | dst;
}

class Tensor {
    Cow<Matrix<uint64_t>> m_;
    Delta<uint64_t> dp_;
    Delta<bool> dm_;
    VersionedMatrix mt_, me_;
    mutable std::atomic<bool> needs_flush{false};

    struct PairHash { size_t operator()(const std::pair<uint64_t, uint64_t> &p) const { return std::hash<uint64_t>()(p.first * 0x9E3779B97F4A7C15ULL ^ p.second); } };

  public:
    Tensor() {}
    Tensor(uint64_t nrows, uint64_t ncols)                       // tensor.rs:244-259
        : m_(Matrix<uint64_t>(nrows, ncols)), dp_(Matrix<uint64_t>(nrows, ncols)), dm_(Matrix<bool>(nrows, ncols)),
          mt_(ncols, nrows), me_(GrB_INDEX_MAX_, GrB_INDEX_MAX_) {}
    Tensor(const Tensor &o) : m_(o.m_), dp_(o.dp_), dm_(o.dm_), mt_(o.mt_), me_(o.me_), needs_flush(o.needs_flush.load()) {}
    Tensor &operator=(const Tensor &o) { m_ = o.m_; dp_ = o.dp_; dm_ = o.dm_; mt_ = o.mt_; me_ = o.me_; needs_flush = o.needs_flush.load(); return *this; }

    const Matrix<uint64_t> &fwd_m() const { return m_.get(); }   // tensor.rs:841-856
    const Matrix<uint64_t> &fwd_dp() const { return dp_.m(); }
    const Matrix<bool> &fwd_dm() const { return dm_.m(); }
    const VersionedMatrix &matrix_t() const { return mt_; }      // tensor.rs:886
    const VersionedMatrix &edge_versioned() const { return me_; }

    void wait_fwd() const {                                      // tensor.rs:268-286
        if (fwd_dp().is_synced() && fwd_dm().is_synced()) return;
        dp_.resync();
        dm_.resync();
        uint64_t base = fwd_m().nvals();
        dp_.latch(dp_.fold_decision(should_fold_read, base));
        dm_.latch(dm_.fold_decision(should_fold_read, base));
    }
    bool eff_get(uint64_t src, uint64_t dst, uint64_t *out) const {  // tensor.rs:290-303
        wait_fwd();
        if (fwd_dp().get(src, dst, out)) return true;
        if (fwd_dm().nvals() != 0 && fwd_dm().contains(src, dst)) return false;
        return fwd_m().get(src, dst, out);
    }
    // edge ids of the pair, ascending (tensor.rs:307-321)
    std::vector<uint64_t> get(uint64_t src, uint64_t dst) const {
        std::vector<uint64_t> ids;
        uint64_t v;
        if (!eff_get(src, dst, &v)) return ids;
        if (v != MULTI_EDGE) { ids.push_back(v); return ids; }
        uint64_t key = compound_key(src, dst);
        auto it = me_.iter(key, key);
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) ids.push_back(std::get<1>(t));
        return ids;
    }
    bool has_multi_edge() const { return me_.nvals() != 0; }
    void wait() const { wait_fwd(); mt_.wait(); me_.wait(); }

    // tensor.rs:333-447
    void set_all_from_slices(const std::vector<uint64_t> &srcs, const std::vector<uint64_t> &dsts, const std::vector<uint64_t> &ids) {
        if (srcs.empty()) return;
        flush();
        fwd_dp().wait();
        fwd_dm().wait();
        bool dm_empty = fwd_dm().nvals() == 0;
        std::unordered_map<std::pair<uint64_t, uint64_t>, size_t, PairHash> batch;
        std::vector<uint64_t> m_srcs, m_dsts, m_ids;
        std::vector<std::pair<bool, uint64_t>> m_masked;
        for (size_t t = 0; t < srcs.size(); t++) {
            uint64_t s = srcs[t], d = dsts[t], id = ids[t];
            uint64_t key = compound_key(s, d);
            auto found = batch.find({s, d});
            if (found != batch.end()) {
                size_t idx = found->second;
                if (idx != SIZE_MAX) {           // second edge of a pair new in this batch: promote the pending slot
                    me_.set(key, m_ids[idx]);
                    m_ids[idx] = MULTI_EDGE;
                    found->second = SIZE_MAX;
                }
                me_.set(key, id);
                continue;
            }
            bool masked = !dm_empty && fwd_dm().contains(s, d);
            uint64_t cur = 0, from_dp_v = 0;
            bool from_dp = fwd_dp().get(s, d, &from_dp_v);
            bool has_cur = from_dp;
            if (from_dp) cur = from_dp_v;
            else if (!masked) has_cur = fwd_m().get(s, d, &cur);
            if (has_cur && cur == MULTI_EDGE) {
                me_.set(key, id);
                batch[{s, d}] = SIZE_MAX;
            } else if (has_cur) {                // present single edge: promote
                me_.set(key, cur);
                me_.set(key, id);
                batch[{s, d}] = SIZE_MAX;
                m_srcs.push_back(s); m_dsts.push_back(d); m_ids.push_back(MULTI_EDGE);
                uint64_t committed = 0;
                bool hc = from_dp && fwd_m().get(s, d, &committed);
                m_masked.push_back({hc, committed});
            } else {                             // first edge of the pair: inline
                batch[{s, d}] = m_ids.size();
                m_srcs.push_back(s); m_dsts.push_back(d); m_ids.push_back(id);
                uint64_t committed = 0;
                bool hc = masked && fwd_m().get(s, d, &committed);
                m_masked.push_back({hc, committed});
            }
        }
        for (size_t i = 0; i < m_srcs.size(); i++) {
            uint64_t s = m_srcs[i], d = m_dsts[i], id = m_ids[i];
            mt_.set(d, s);
            if (m_masked[i].first) {
                dm_.erase(s, d);
                if (m_masked[i].second == id) { dp_.erase(s, d); continue; }   // deltas cancel: committed value restored
            }
            dp_.insert(s, d, id);
        }
    }

    // tensor.rs:454-629.  rels = (edge_id, src, dst); returns the pairs that lost their last edge.
    std::vector<std::pair<uint64_t, uint64_t>> remove_all(const std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> &rels) {
        std::vector<std::pair<uint64_t, uint64_t>> emptied;
        if (rels.empty()) return emptied;
        flush();
        if (!has_multi_edge()) return remove_bulk(rels);
        wait_fwd();
        enum Kind { Multi, Single, Emptied, Absent };
        struct Plan { Kind kind; std::vector<uint64_t> ids; uint64_t id = 0; bool demoted = false; };
        std::map<std::pair<uint64_t, uint64_t>, Plan> plans;
        std::vector<std::pair<uint64_t, uint64_t>> me_del;
        for (auto &rel : rels) {
            uint64_t id = std::get<0>(rel), src = std::get<1>(rel), dst = std::get<2>(rel);
            uint64_t key = compound_key(src, dst);
            auto it = plans.find({src, dst});
            if (it == plans.end()) {
                Plan p;
                uint64_t v;
                if (!eff_get(src, dst, &v)) p.kind = Absent;
                else if (v == MULTI_EDGE) {
                    p.kind = Multi;
                    auto mi = me_.iter(key, key);
                    std::tuple<uint64_t, uint64_t> t;
                    while (mi.next(t)) p.ids.push_back(std::get<1>(t));
                } else { p.kind = Single; p.id = v; }
                it = plans.emplace(std::make_pair(src, dst), p).first;
            }
            Plan &p = it->second;
            if (p.kind == Multi) {
                auto pos = std::lower_bound(p.ids.begin(), p.ids.end(), id);
                if (pos == p.ids.end() || *pos != id) continue;
                p.ids.erase(pos);
                me_del.push_back({key, id});
                if (p.ids.size() == 1) {         // down to one edge: demote
                    uint64_t last = p.ids[0];
                    me_del.push_back({key, last});
                    p.kind = Single; p.id = last; p.demoted = true; p.ids.clear();
                }
            } else if (p.kind == Single && p.id == id) {
                p.kind = Emptied;
                emptied.push_back({src, dst});
            }
        }
        for (auto &d : me_del) me_.remove(d.first, d.second);
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> dp_set;
        for (auto &kv : plans) {
            uint64_t src = kv.first.first, dst = kv.first.second;
            const Plan &p = kv.second;
            if (p.kind == Emptied) {
                dp_.erase(src, dst);
                if (fwd_m().contains(src, dst)) dm_.insert(src, dst);
                mt_.remove(dst, src);
            } else if (p.kind == Single && p.demoted) {
                uint64_t committed;
                if (fwd_m().get(src, dst, &committed) && committed == p.id) dp_.erase(src, dst);
                else dp_set.push_back(std::make_tuple(src, dst, p.id));
            }
        }
        for (auto &t : dp_set) dp_.insert(std::get<0>(t), std::get<1>(t), std::get<2>(t));
        return emptied;
    }

    // remove_all's fast path when no pair has several edges: a few bulk GraphBLAS ops (same math as remove_mask).  Every named
    // pair is removed and reported, whatever id names it.
    std::vector<std::pair<uint64_t, uint64_t>> remove_bulk(const std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> &rels) {
        std::vector<std::pair<uint64_t, uint64_t>> emptied;
        wait_fwd();
        uint64_t nr = fwd_m().nrows(), nc = fwd_m().ncols();
        std::vector<uint64_t> mr, mc, tr, tc;
        for (auto &r : rels) { mr.push_back(std::get<1>(r)); mc.push_back(std::get<2>(r)); tr.push_back(std::get<2>(r)); tc.push_back(std::get<1>(r)); }
        Matrix<bool> m_mask(nr, nc), mt_mask(nc, nr);
        m_mask.build(mr, mc);
        mt_mask.build(tr, tc);
        dm_.tombstone_masked(m_mask, fwd_m());   // PAIR never reads m's u64 values: edge id 0 is safe
        dp_.remove_all(m_mask);
        mt_.remove_mask(mt_mask);
        for (auto &r : rels) emptied.push_back({std::get<1>(r), std::get<2>(r)});
        return emptied;
    }

    // the nine layer handles (B200_TensorLayers order), borrowed
    B200_TensorLayers layers() const {
        return B200_TensorLayers{fwd_m().inner(), fwd_dp().inner(), fwd_dm().inner(), mt_.m().inner(), mt_.dp().inner(), mt_.dm().inner(),
                                 me_.m().inner(), me_.dp().inner(), me_.dm().inner()};
    }
    // layers() once every layer's pending work is applied, as B200_expand_edges and B200_var_len_trails read them
    B200_TensorLayers waited_layers() const {
        wait();
        fwd_m().wait(); fwd_dp().wait(); fwd_dm().wait();
        mt_.wait_all(); me_.wait_all();
        return layers();
    }
    // the six Delta counters: dp, dm, mt's dp, dm, me's dp, dm
    void counts(uint64_t *out6) const {
        out6[0] = dp_.get_count(); out6[1] = dm_.get_count();
        mt_.counts(out6 + 2);
        me_.counts(out6 + 4);
    }

    // set_all_from_slices with its read phase as one device call (B200_Tensor_insert_plan): the plan replaces every dp.get /
    // dm.contains / m.get / mt.m / me.m probe, so a base with no host form is never downloaded.  The write phase makes the
    // reference's Delta calls, in number and, where the order can change a counter, in order.
    void set_all_from_slices_dev(const std::vector<uint64_t> &srcs, const std::vector<uint64_t> &dsts, const std::vector<uint64_t> &ids) {
        if (srcs.empty()) return;
        if (srcs.size() != dsts.size() || srcs.size() != ids.size()) throw std::logic_error("set_all_from_slices_dev: slices differ in length");
        flush();
        fwd_dp().wait();
        fwd_dm().wait();
        const size_t n = srcs.size();
        std::vector<uint64_t> in_src(n), in_dst(n), in_val(n), me_key(2 * n), me_id(2 * n);
        std::vector<uint8_t> in_flags(n), me_base(2 * n);
        uint64_t nin = 0, nme = 0;
        B200_TensorLayers L = layers();
        grb_ok(B200_Tensor_insert_plan(&L, srcs.data(), dsts.data(), ids.data(), n, in_src.data(), in_dst.data(), in_val.data(),
                                       in_flags.data(), &nin, me_key.data(), me_id.data(), me_base.data(), &nme),
               "B200_Tensor_insert_plan");
        for (uint64_t k = 0; k < nme; k++) me_.set_known(me_key[k], me_id[k], me_base[k] != 0);
        // dp takes inserts and (CANCEL) erases of absent entries.  Its counter saturates at 0, so when the erases could reach 0 the
        // records go in the reference's order, the batch order of each pair's first edge; every other layer takes one kind of call
        // and any order gives the same counter.
        std::vector<uint64_t> order(nin);
        for (uint64_t k = 0; k < nin; k++) order[k] = k;
        uint64_t cancels = 0;
        for (uint64_t k = 0; k < nin; k++) cancels += (in_flags[k] & B200_PLAN_CANCEL) != 0;
        if (cancels > dp_.get_count()) {
            std::unordered_map<uint64_t, uint64_t> first;
            for (size_t t = n; t-- > 0;) first[compound_key(srcs[t], dsts[t])] = t;
            std::sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) {
                return first[compound_key(in_src[a], in_dst[a])] < first[compound_key(in_src[b], in_dst[b])];
            });
        }
        for (uint64_t k : order) {
            const uint64_t s = in_src[k], d = in_dst[k], id = in_val[k];
            const uint8_t f = in_flags[k];
            mt_.set_known(d, s, (f & B200_PLAN_MT_BASE) != 0);
            if (f & B200_PLAN_COMMITTED) {
                dm_.erase(s, d);
                if (f & B200_PLAN_CANCEL) { dp_.erase(s, d); continue; }
            }
            dp_.insert(s, d, id);
        }
    }

    // remove_all with its read phase as one device call (B200_Tensor_remove_plan).  Without multi-edges it keeps remove_all's bulk
    // path, which removes a named pair whatever id names it.  Emptied pairs come back ascending (the reference: discovery order).
    std::vector<std::pair<uint64_t, uint64_t>> remove_all_dev(const std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> &rels) {
        std::vector<std::pair<uint64_t, uint64_t>> emptied;
        if (rels.empty()) return emptied;
        flush();
        if (!has_multi_edge()) return remove_bulk(rels);
        wait_fwd();
        const size_t n = rels.size();
        std::vector<uint64_t> rid(n), rs(n), rd(n);
        for (size_t k = 0; k < n; k++) { rid[k] = std::get<0>(rels[k]); rs[k] = std::get<1>(rels[k]); rd[k] = std::get<2>(rels[k]); }
        std::vector<uint64_t> pr_src(n), pr_dst(n), pr_val(n), me_key(2 * n), me_id(2 * n);
        std::vector<uint8_t> pr_flags(n), me_base(2 * n);
        uint64_t npr = 0, nme = 0;
        B200_TensorLayers L = layers();
        grb_ok(B200_Tensor_remove_plan(&L, rid.data(), rs.data(), rd.data(), n, pr_src.data(), pr_dst.data(), pr_val.data(),
                                       pr_flags.data(), &npr, me_key.data(), me_id.data(), me_base.data(), &nme),
               "B200_Tensor_remove_plan");
        for (uint64_t k = 0; k < nme; k++) me_.remove_known(me_key[k], me_id[k], me_base[k] != 0);
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> dp_set;
        for (uint64_t k = 0; k < npr; k++) {                     // pairs ascending, as remove_all's std::map walk
            const uint64_t src = pr_src[k], dst = pr_dst[k];
            const uint8_t f = pr_flags[k];
            if (f & B200_PLAN_EMPTIED) {
                dp_.erase(src, dst);
                if (f & B200_PLAN_M_HAS) dm_.insert(src, dst);
                mt_.remove_known(dst, src, (f & B200_PLAN_MT_BASE) != 0);
                emptied.push_back({src, dst});
            } else if (f & B200_PLAN_M_EQ) {
                dp_.erase(src, dst);
            } else {
                dp_set.push_back(std::make_tuple(src, dst, pr_val[k]));
            }
        }
        for (auto &t : dp_set) dp_.insert(std::get<0>(t), std::get<1>(t), std::get<2>(t));
        return emptied;
    }

    void flush() {                                               // tensor.rs:702-751
        if (needs_flush.load(std::memory_order_relaxed)) {
            fwd_m().wait(); fwd_dp().wait(); fwd_dm().wait();
            bool fold_dp = dp_.take_fold(), fold_dm = dm_.take_fold();
            if (fold_dp || fold_dm) {
                uint64_t nr = fwd_m().nrows(), nc = fwd_m().ncols();
                Matrix<uint64_t> new_m(nr, nc);
                if (fold_dp && fold_dm) new_m.element_wise_add<uint64_t>(&fwd_dm(), &fwd_m(), &fwd_dp(), Descriptor::RC); // SECOND: dp wins
                else if (fold_dp) new_m.element_wise_add<uint64_t>(nullptr, &fwd_m(), &fwd_dp());
                else new_m.select(fwd_dm(), fwd_m());
                new_m.wait();
                m_.replace(new_m);
                if (fold_dp) dp_.clear(nr, nc);
                if (fold_dm) dm_.clear(nr, nc);
            }
            needs_flush.store(false, std::memory_order_relaxed);
        }
        mt_.flush();
        me_.flush();
    }
    void fold_latched() {                                        // tensor.rs:757-765
        wait_fwd();
        if (dp_.folding() || dm_.folding()) { needs_flush = true; flush(); }
        mt_.fold_latched();
        me_.fold_latched();
    }
    void fold_oversized() {                                      // tensor.rs:773-788
        uint64_t base = fwd_m().nvals();
        bool odp = delta_dominates_base(dp_.get_count(), base), odm = delta_dominates_base(dm_.get_count(), base);
        if (odp || odm) { dp_.latch(odp); dm_.latch(odm); needs_flush = true; flush(); }
        mt_.fold_oversized();
        me_.fold_oversized();
    }
    Matrix<bool> extract() const {                               // tensor.rs:793-804
        wait_fwd();
        Matrix<bool> out(fwd_m().nrows(), fwd_m().ncols());
        out.set_pattern<uint64_t>(nullptr, fwd_m());
        if (fwd_dm().nvals() > 0) out.remove_all(fwd_dm());
        if (fwd_dp().nvals() > 0) out.set_pattern<uint64_t>(nullptr, fwd_dp());
        return out;
    }
    void rebuild_backward() { mt_ = VersionedMatrix::from_matrix(extract().transpose()); }  // tensor.rs:814-816
    Tensor dup() const {                                         // tensor.rs:825-838
        uint64_t base = fwd_m().nvals();
        bool fdp = dp_.fold_decision(should_fold, base), fdm = dm_.fold_decision(should_fold, base);
        Tensor t;
        t.m_ = m_.new_version();
        t.dp_ = dp_.new_version(fdp);
        t.dm_ = dm_.new_version(fdm);
        t.mt_ = mt_.dup();
        t.me_ = me_.dup();
        t.needs_flush = fdp || fdm;
        return t;
    }
    LayerIter<uint64_t> fwd_iter(uint64_t min_row = 0, uint64_t max_row = UINT64_MAX) const {   // tensor.rs:873-882
        wait_fwd();
        return LayerIter<uint64_t>(fwd_m(), fwd_dp(), fwd_dm(), min_row, max_row);
    }
    uint64_t multi_pairs() const {                               // tensor.rs:980-1003
        if (me_.nvals() == 0) return 0;
        me_.wait();
        if (me_.dp().nvals() == 0 && me_.dm().nvals() == 0) {
            int64_t k = me_.m().hyper_vector_count();
            if (k >= 0) return (uint64_t)k;
        }
        uint64_t rows = 0, last = UINT64_MAX;
        bool have = false;
        auto it = me_.iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) if (!have || std::get<0>(t) != last) { rows++; last = std::get<0>(t); have = true; }
        return rows;
    }
    uint64_t edge_count() const {                                // tensor.rs:903-913
        wait_fwd();
        uint64_t shadow = fwd_dp().nvals() == 0 ? 0 : fwd_dp().intersection_nvals(fwd_m());
        return fwd_m().nvals() + fwd_dp().nvals() - fwd_dm().nvals() - shadow - multi_pairs() + me_.nvals();
    }
    // ---- the C-compatible RDB form (tensor.rs:1049-1204) ----
    // Forward matrix as UINT64: a single-edge pair stores its edge id (MSB clear), a multi-edge pair stores (edge count | MSB) and
    // its id list follows in the tensor section as a BOOL vector of size GrB_INDEX_MAX whose INDICES are the ids.  Deltas are
    // folded into the base on the way out (two empty layers follow), then total edge count, then two groups (base, delta-plus).
    static const uint64_t MSB_MASK = (uint64_t)1 << 63;
    void encode(Stream &w) const {                               // tensor.rs:1053-1126
        uint64_t nrows = fwd_m().nrows(), ncols = fwd_m().ncols();
        Matrix<uint64_t> fm(nrows, ncols), empty(nrows, ncols);
        std::vector<std::tuple<uint64_t, uint64_t, std::vector<uint64_t>>> multi;
        {
            auto it = fwd_iter(0, UINT64_MAX);
            std::tuple<uint64_t, uint64_t, uint64_t> t;
            while (it.next(t)) {
                uint64_t src = std::get<0>(t), dst = std::get<1>(t), inl = std::get<2>(t);
                if (inl == MULTI_EDGE) {
                    std::vector<uint64_t> ids;
                    uint64_t key = compound_key(src, dst);
                    auto mi = me_.iter(key, key);
                    std::tuple<uint64_t, uint64_t> e;
                    while (mi.next(e)) ids.push_back(std::get<1>(e));
                    fm.set(src, dst, (uint64_t)ids.size() | MSB_MASK);
                    multi.push_back(std::make_tuple(src, dst, std::move(ids)));
                } else {
                    fm.set(src, dst, inl);
                }
            }
        }
        // the reference collects the triples and calls build(); here they are set one by one and assembled on the host by wait():
        // the container unload that follows needs the host form anyway, so nothing of this visits the device
        fm.wait();
        encode_matrix(fm, w);
        encode_matrix(empty, w);      // delta-plus
        encode_matrix(empty, w);      // delta-minus
        uint64_t total = edge_count();
        w.write_unsigned(total);
        if (total == 0) return;
        w.write_unsigned((uint64_t)multi.size());
        for (auto &mp : multi) {
            w.write_unsigned(std::get<0>(mp));
            w.write_unsigned(std::get<1>(mp));
            encode_id_blob(std::get<2>(mp), GrB_INDEX_MAX_, w);
        }
        w.write_unsigned(0);          // empty delta-plus tensor group
    }
    // The backward matrix is left empty: the caller rebuilds it (rebuild_backward) after decode, as in the reference.
    static Tensor decode(Stream &r) {                            // tensor.rs:1130-1204
        Matrix<uint64_t> fwd_m = decode_matrix<uint64_t>(r), fwd_dp = decode_matrix<uint64_t>(r);
        Matrix<bool> fwd_dm = decode_matrix<bool>(r);
        uint64_t nrows = fwd_m.nrows(), ncols = fwd_m.ncols();
        Matrix<uint64_t> m(nrows, ncols);
        VersionedMatrix me(GrB_INDEX_MAX_, GrB_INDEX_MAX_);
        bool dm_empty = fwd_dm.nvals() == 0;
        std::tuple<uint64_t, uint64_t, uint64_t> t;
        {
            auto it = fwd_m.iter(0, UINT64_MAX);
            while (it.next(t)) {
                uint64_t src = std::get<0>(t), dst = std::get<1>(t), value = std::get<2>(t);
                if (!dm_empty && fwd_dm.contains(src, dst)) continue;      // deleted (a live replacement id lives in fwd_dp)
                m.set(src, dst, (value & MSB_MASK) == 0 ? value : MULTI_EDGE);
            }
        }
        {
            auto it = fwd_dp.iter(0, UINT64_MAX);
            while (it.next(t)) m.set(std::get<0>(t), std::get<1>(t), (std::get<2>(t) & MSB_MASK) == 0 ? std::get<2>(t) : MULTI_EDGE);
        }
        uint64_t total_tensor_count = r.read_unsigned();
        if (total_tensor_count > 0) {
            for (int group = 0; group < 2; group++) {            // base (TM), then delta-plus (TDP)
                uint64_t count = r.read_unsigned();
                for (uint64_t k = 0; k < count; k++) {
                    uint64_t src = r.read_unsigned(), dst = r.read_unsigned();
                    uint64_t key = compound_key(src, dst);
                    for (uint64_t edge_id : decode_id_blob(r)) me.set(key, edge_id);
                }
            }
        }
        m.wait();
        Tensor out(nrows, ncols);
        out.m_ = Cow<Matrix<uint64_t>>(m);
        out.mt_ = VersionedMatrix(0, 0);
        out.me_ = me;
        return out;
    }

    // GRAPH.BULK's edge load into an empty tensor (bulk_insert.rs:497 -> graph.rs:2062-2135) through the device-side build
    // B200_Tensor_bulk_build: the state Tensor::new + set_all_from_slices + the end-of-command fold would reach, in one call
    static Tensor bulk_load(uint64_t nrows, uint64_t ncols, const std::vector<uint64_t> &srcs, const std::vector<uint64_t> &dsts,
                            const std::vector<uint64_t> &ids) {
        if (srcs.size() != dsts.size() || srcs.size() != ids.size()) throw std::logic_error("bulk_load: slices differ in length");
        GrB_Matrix raw = nullptr;
        GrB_Index *mk = nullptr, *mi = nullptr, nm = 0;
        grb_ok(B200_Tensor_bulk_build(&raw, &mk, &mi, &nm, nrows, ncols, srcs.data(), dsts.data(), ids.data(), srcs.size()),
               "B200_Tensor_bulk_build");
        Tensor t(nrows, ncols);
        t.m_ = Cow<Matrix<uint64_t>>(Matrix<uint64_t>::adopt(raw, false));
        if (nm) {
            std::vector<uint64_t> keys(mk, mk + nm), eids(mi, mi + nm);
            std::free(mk);
            std::free(mi);
            Matrix<bool> me(GrB_INDEX_MAX_, GrB_INDEX_MAX_);
            me.build(keys, eids);
            me.wait();
            t.me_ = VersionedMatrix::from_matrix(me);
        }
        t.rebuild_backward();
        return t;
    }

    // every (src, dst, edge_id): inline singles first, then the multi-edge ids (tensor.rs:921-936)
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> iter_edges() const {
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> out;
        auto it = fwd_iter();
        std::tuple<uint64_t, uint64_t, uint64_t> t;
        while (it.next(t)) if (std::get<2>(t) != MULTI_EDGE) out.push_back(t);
        if (me_.nvals() != 0) {
            auto mi = me_.iter(0, GrB_INDEX_MAX_);
            std::tuple<uint64_t, uint64_t> e;
            while (mi.next(e)) out.push_back(std::make_tuple(std::get<0>(e) >> 32, std::get<0>(e) & 0xFFFFFFFFULL, std::get<1>(e)));
        }
        return out;
    }
};

} // namespace fdb
