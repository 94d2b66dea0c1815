// cond_traverse.hpp -- C++ mirror of the batched F*A path of the reference's CondTraverse operator
// (graph/src/runtime/ops/cond_traverse.rs:452-751), reduced to what sits on the GraphBLAS boundary:
//   collect (row_i, src) + source-label pre-filter   :554-589
//   F = Matrix<bool>(|batch|, n); F.build(rows, srcs) :600-601
//   for hop: delta_lmxm_into(F)                        :602-605   (matrix.rs:1317-1402)
//   F.wait(); for (row_i, dest) in F.iter()            :608, 644
//   destination-label post-filter                      :646-652
// Batch/column plumbing (gather, set_column, null padding) is runtime code outside the hot path (SURVEY 2, #17).
#pragma once
#include "tensor.hpp"

namespace fdb {

// Graph::node_has_label_id (graph.rs:1057-1065): label matrices are n x n diagonal (graph.rs:1191)
inline bool node_has_label(const VersionedMatrix &label, uint64_t id) { return label.get(id, id); }

struct ExpandResult {
    std::vector<uint64_t> row_idx; // index into the input batch (active_subset position)
    std::vector<uint64_t> dest;    // destination node id
};

static const size_t BATCH_SIZE = 1024; // graph/src/runtime/batch.rs:81

// Graph::build_relationship_matrix_unrestricted (graph.rs:2520-2550), statement for statement: the exact union of several
// relationship types' forward layers, U_t (m_t \ dm_t) u dp_t, as a fresh delta-free matrix.  set_pattern has no replace, so an
// entry an earlier type contributed survives a later type's dm.  What CondTraverseOp multiplies by for -[:R1|R2]-> before the
// union hop; tests compare the union hop against it.
inline VersionedMatrix union_by_extract(const std::vector<const Tensor *> &types) {
    Matrix<bool> m = types[0]->extract();
    for (size_t k = 1; k < types.size(); k++) {
        const Tensor *t = types[k];
        t->wait_fwd();
        m.set_pattern<uint64_t>(&t->fwd_dm(), t->fwd_m(), Descriptor::C);
        m.set_pattern<uint64_t>(nullptr, t->fwd_dp());
    }
    return VersionedMatrix::from_matrix(m);
}

// TraversalMatrix (cond_traverse.rs:64-90): the adjacency VersionedMatrix<bool>, one relationship type's Tensor, or several types'
// Tensors (-[:R1|R2]->, cond_traverse.rs:493, 523): the union hop over their forward layers (B200_Matrix_union_lmxm) in place of
// the reference's build_relationship_matrix_unrestricted plus a hop by the fresh matrix.  A one-type list is still a union hop.
struct TraversalMatrix {
    const VersionedMatrix *vm = nullptr;
    const Tensor *t = nullptr;
    std::vector<const Tensor *> ts;
    TraversalMatrix(const VersionedMatrix *v) : vm(v) {}
    TraversalMatrix(const Tensor *x) : t(x) {}
    TraversalMatrix(std::vector<const Tensor *> xs) : ts(std::move(xs)) {
        if (ts.empty()) throw std::invalid_argument("TraversalMatrix: a multi-type hop needs at least one type");
    }
    bool is_union() const { return !ts.empty(); }
    uint64_t ncols() const { return vm ? vm->ncols() : (t ? t : ts[0])->fwd_m().ncols(); }
    void delta_lmxm_into(Matrix<bool> &f) const {                // cond_traverse.rs:77-85
        if (vm) f.delta_lmxm(vm->m(), vm->dp(), vm->dm());
        else if (t) f.delta_lmxm(t->fwd_m(), t->fwd_dp(), t->fwd_dm());
        else {
            std::vector<GrB_Matrix> m, dp, dm;
            operands(m, dp, dm);
            f.union_lmxm(m, dp, dm);
        }
    }
    // the (m, dp, dm) handles delta_lmxm_into multiplies by, appended: one triple, or one per type of a union hop
    void operands(std::vector<GrB_Matrix> &m, std::vector<GrB_Matrix> &dp, std::vector<GrB_Matrix> &dm) const {
        if (vm) {
            vm->dp().wait(); vm->dm().wait();
            m.push_back(vm->m().inner()); dp.push_back(vm->dp().inner()); dm.push_back(vm->dm().inner());
            return;
        }
        if (t) {
            t->fwd_dp().wait(); t->fwd_dm().wait();
            m.push_back(t->fwd_m().inner()); dp.push_back(t->fwd_dp().inner()); dm.push_back(t->fwd_dm().inner());
            return;
        }
        for (const Tensor *x : ts) {                             // as build_relationship_matrix_unrestricted: wait_fwd per type
            x->wait_fwd();
            x->fwd_m().wait(); x->fwd_dp().wait(); x->fwd_dm().wait();
            m.push_back(x->fwd_m().inner()); dp.push_back(x->fwd_dp().inner()); dm.push_back(x->fwd_dm().inner());
        }
    }
};

// Every hop of a batch in one library call (CSR hand-off): (row, dest) pairs of F * hops, in ascending order.  The batch rows are
// the surviving sources' positions in the input batch.  Hops of one operand each go to B200_traverse_batch_delta; with a union hop
// among them the hop groups go to B200_traverse_batch_union.
inline void traverse_coalesced(const std::vector<uint64_t> &rows, const std::vector<uint64_t> &srcs,
                               const std::vector<TraversalMatrix> &hops, std::vector<uint64_t> &out_row, std::vector<uint64_t> &out_dest) {
    std::vector<GrB_Matrix> m, dp, dm;
    std::vector<int> nops, uni;
    bool any_union = false;
    for (const TraversalMatrix &h : hops) {
        const size_t before = m.size();
        h.operands(m, dp, dm);
        nops.push_back((int)(m.size() - before));
        uni.push_back(h.is_union() ? 1 : 0);
        any_union = any_union || h.is_union();
    }
    std::vector<uint64_t> p(srcs.size() + 1);
    std::vector<uint32_t> j(std::max<size_t>(1024, 16 * srcs.size()));
    uint64_t nv = 0;
    for (int attempt = 0; attempt < 2; attempt++) {              // a result larger than the first guess is rerun into its size
        GrB_Info info = any_union
            ? B200_traverse_batch_union(srcs.data(), srcs.size(), nops.data(), uni.data(), (int)hops.size(), m.data(), dp.data(),
                                        dm.data(), B200_OUT_CSR, nullptr, 0, p.data(), j.data(), j.size(), &nv, nullptr, nullptr)
            : B200_traverse_batch_delta(srcs.data(), srcs.size(), m.data(), dp.data(), dm.data(), (int)hops.size(),
                                        B200_OUT_CSR, nullptr, 0, p.data(), j.data(), j.size(), &nv, nullptr, nullptr);
        if (info == GrB_INSUFFICIENT_SPACE && attempt == 0) { j.resize(nv); continue; }
        grb_ok(info, any_union ? "B200_traverse_batch_union" : "B200_traverse_batch_delta");
        break;
    }
    for (size_t r = 0; r < srcs.size(); r++)
        for (uint64_t q = p[r]; q < p[r + 1]; q++) { out_row.push_back(rows[r]); out_dest.push_back(j[q]); }
}

// ---- relationship ids: named-edge, incoming and bidirectional hops (B200_expand_edges) ----
// Row i of a batch covers p[i] .. p[i+1]: the neighbour, the edge id, the type index and whether the entry belongs to the reverse
// block; forward block first, inside a block neighbour, type index, id ascending.
struct EdgeExpansion {
    std::vector<uint64_t> p{0};
    std::vector<uint32_t> node;
    std::vector<uint64_t> edge;
    std::vector<uint16_t> type;
    std::vector<uint8_t> rev;
    void push(uint64_t d, uint64_t id, size_t t, bool r) { node.push_back((uint32_t)d); edge.push_back(id); type.push_back((uint16_t)t); rev.push_back(r); }
    void end_row() { p.push_back(edge.size()); }
};

// every row's relationships in one library call, each type's layers passed after Tensor::wait()
inline EdgeExpansion expand_edges(const std::vector<uint64_t> &srcs, const std::vector<uint64_t> *targets,
                                  const std::vector<const Tensor *> &types, int dir, int mode) {
    std::vector<B200_TensorLayers> ls;
    for (const Tensor *t : types) ls.push_back(t->waited_layers());
    EdgeExpansion r;
    const size_t n = srcs.size();
    r.p.assign(n + 1, 0);
    r.node.resize(std::max<size_t>(1024, 4 * n));
    uint64_t nv = 0;
    for (int attempt = 0; attempt < 2; attempt++) {              // a result larger than the first guess is rerun into its size
        r.edge.resize(r.node.size()); r.type.resize(r.node.size()); r.rev.resize(r.node.size());
        GrB_Info info = B200_expand_edges(srcs.data(), targets ? targets->data() : nullptr, n, ls.data(), (int)ls.size(), dir, mode,
                                          r.p.data(), r.node.data(), r.edge.data(), r.type.data(), r.rev.data(), r.node.size(), &nv);
        if (info == GrB_INSUFFICIENT_SPACE && attempt == 0) { r.node.resize(nv); continue; }
        grb_ok(info, "B200_expand_edges");
        break;
    }
    r.node.resize(nv); r.edge.resize(nv); r.type.resize(nv); r.rev.resize(nv);
    return r;
}

// process_pairs' edge loop for one (src, dst) pair of a block (cond_traverse.rs:1084-1113 emit_relationship, :676-687 bind_edge):
// the pair's ids per type in edge_type_indices order, all of them or the first
inline void emit_pair_edges(const std::vector<const Tensor *> &types, uint64_t src, uint64_t dst, uint64_t nbr, bool rev, bool first,
                            EdgeExpansion &r) {
    for (size_t t = 0; t < types.size(); t++) {
        for (uint64_t id : types[t]->get(src, dst)) {
            r.push(nbr, id, t, rev);
            if (first) return;
        }
    }
}

// the neighbours a seeked structural iterator over the types yields for `row`, ascending: the forward layers (fwd_iter) or the
// maintained transpose (build_transposed_iter, cond_traverse.rs:221-235)
inline std::vector<uint64_t> row_neighbours(const std::vector<const Tensor *> &types, uint64_t row, bool transposed) {
    std::vector<uint64_t> out;
    for (const Tensor *t : types) {
        if (transposed) {
            auto it = t->matrix_t().iter(row, row);
            std::tuple<uint64_t, uint64_t> e;
            while (it.next(e)) out.push_back(std::get<1>(e));
        } else {
            auto it = t->fwd_iter(row, row);
            std::tuple<uint64_t, uint64_t, uint64_t> e;
            while (it.next(e)) out.push_back(std::get<1>(e));
        }
    }
    std::sort(out.begin(), out.end());
    out.erase(std::unique(out.begin(), out.end()), out.end());
    return out;
}

// expand_row's edge loops restated statement for statement (cond_traverse.rs:844-935): forward pairs from the structural iterator
// seeked at the source, reverse pairs from matrix_t()'s iterator (self-loops skipped under BOTH), ids by Tensor::get.  The route
// B200_expand_edges replaces; tests compare against it.
inline EdgeExpansion expand_edges_by_get(const std::vector<uint64_t> &srcs, const std::vector<const Tensor *> &types, int dir, int mode) {
    EdgeExpansion r;
    const bool first = mode == B200_EDGES_FIRST;
    for (uint64_t s : srcs) {
        if (dir != B200_DIR_IN)
            for (uint64_t d : row_neighbours(types, s, false)) emit_pair_edges(types, s, d, d, false, first, r);
        if (dir != B200_DIR_OUT)
            for (uint64_t k : row_neighbours(types, s, true)) {
                if (dir == B200_DIR_BOTH && k == s) continue;
                emit_pair_edges(types, k, s, k, true, first, r);
            }
        r.end_row();
    }
    return r;
}

// ExpandInto with the edge bound (expand_into.rs:121-258): Tensor::get on (src, dst), and under BOTH on (dst, src) when they differ
inline EdgeExpansion expand_into_by_get(const std::vector<uint64_t> &srcs, const std::vector<uint64_t> &dsts,
                                        const std::vector<const Tensor *> &types, int dir, int mode) {
    EdgeExpansion r;
    const bool first = mode == B200_EDGES_FIRST;
    for (size_t i = 0; i < srcs.size(); i++) {
        const uint64_t s = srcs[i], d = dsts[i];
        if (dir != B200_DIR_IN) emit_pair_edges(types, s, d, d, false, first, r);
        if (dir == B200_DIR_IN || (dir == B200_DIR_BOTH && d != s)) emit_pair_edges(types, d, s, d, true, first, r);
        r.end_row();
    }
    return r;
}

// today's bind_edge route on the batched path (cond_traverse.rs:600-608, 663-702): the (row, dest) pairs of one union hop over
// the types (B200_traverse_batch_union), then one Tensor::get per pair for its first id
inline EdgeExpansion bind_edge_after_traverse(const std::vector<uint64_t> &srcs, const std::vector<const Tensor *> &types) {
    std::vector<uint64_t> rows(srcs.size()), out_row, out_dest;
    for (size_t i = 0; i < rows.size(); i++) rows[i] = i;
    traverse_coalesced(rows, srcs, {TraversalMatrix(types)}, out_row, out_dest);
    EdgeExpansion r;
    size_t q = 0;
    for (size_t i = 0; i < srcs.size(); i++) {
        for (; q < out_row.size() && out_row[q] == i; q++) emit_pair_edges(types, srcs[i], out_dest[q], out_dest[q], false, true, r);
        r.end_row();
    }
    return r;
}

// fuse_dst_labels (SURVEY 8f-2): label matrices are diagonal (graph.rs:1191), so the destination filter F*A*L_dst
// (graph.rs:2600-2626) is one more delta_lmxm against the label's VersionedMatrix -- a column filter in frontier form on
// the device -- instead of a node_has_label probe (1-3 extractElement calls) per output pair on the host.
// coalesced: every hop, clean or dirty, and every fused label hop go to the library in ONE call (traverse_coalesced) instead of a
// delta_lmxm per hop; the same pairs come back.
inline ExpandResult expand_batch(const std::vector<uint64_t> &src_ids, const std::vector<TraversalMatrix> &hops,
                                 const std::vector<const VersionedMatrix *> &src_labels,
                                 const std::vector<const VersionedMatrix *> &dst_labels, bool fuse_dst_labels = false,
                                 bool coalesced = false) {
    ExpandResult out;
    if (hops.empty() || src_ids.empty()) return out;
    uint64_t ncols = hops[0].ncols();
    std::vector<uint64_t> row_idx_buf, col_idx_buf;
    row_idx_buf.reserve(src_ids.size());
    col_idx_buf.reserve(src_ids.size());
    for (size_t i = 0; i < src_ids.size(); i++) {
        bool ok = true;
        for (const VersionedMatrix *l : src_labels) if (!node_has_label(*l, src_ids[i])) { ok = false; break; }
        if (!ok) continue;                       // pre-filter src by label (= L_src * F)
        row_idx_buf.push_back((uint64_t)i);
        col_idx_buf.push_back(src_ids[i]);
    }
    if (row_idx_buf.empty()) return out;
    if (coalesced) {
        std::vector<TraversalMatrix> all(hops);
        if (fuse_dst_labels)
            for (const VersionedMatrix *l : dst_labels) all.push_back(TraversalMatrix(l));
        std::vector<uint64_t> rows, dests;
        traverse_coalesced(row_idx_buf, col_idx_buf, all, rows, dests);
        for (size_t k = 0; k < dests.size(); k++) {
            bool ok = true;
            if (!fuse_dst_labels)
                for (const VersionedMatrix *l : dst_labels) if (!node_has_label(*l, dests[k])) { ok = false; break; }
            if (!ok) continue;                   // post-filter final-hop dst label (= F * A * R_dst)
            out.row_idx.push_back(rows[k]);
            out.dest.push_back(dests[k]);
        }
        return out;
    }
    Matrix<bool> f(src_ids.size(), ncols);
    f.build(row_idx_buf, col_idx_buf);
    for (const TraversalMatrix &h : hops) h.delta_lmxm_into(f);
    if (fuse_dst_labels)
        for (const VersionedMatrix *l : dst_labels) TraversalMatrix(l).delta_lmxm_into(f);
    f.wait();                                    // flush pending mxm work before attaching the row iterator
    auto it = f.iter(0, UINT64_MAX);
    std::tuple<uint64_t, uint64_t> t;
    while (it.next(t)) {
        uint64_t dest = std::get<1>(t);
        bool ok = true;
        if (!fuse_dst_labels)
            for (const VersionedMatrix *l : dst_labels) if (!node_has_label(*l, dest)) { ok = false; break; }
        if (!ok) continue;                       // post-filter final-hop dst label (= F * A * R_dst)
        out.row_idx.push_back(std::get<0>(t));
        out.dest.push_back(dest);
    }
    return out;
}

// The batch boundary on the way out (graph/src/runtime/batch.rs:81, 274-287, 832): the (parent row, destination) pairs leave the
// operator re-packed into batches of <= BATCH_SIZE rows -- a `Column::NodeIds` with the destinations plus a selection vector
// (`Vec<u16>`: index of the parent row in the INPUT batch) that `Batch::gather` uses to copy the parent's columns next to it.
// Pairs arrive in ascending (row, dest) order (the iterator contract), so every output batch is a contiguous, ordered slice.
struct OutBatch {
    std::vector<uint64_t> node_ids;    // Column::NodeIds(Vec<NodeId>)  (graph.rs:139: NodeId(u64))
    std::vector<uint16_t> selection;   // parent row per output row; input batches hold <= BATCH_SIZE rows, so u16 suffices
};
inline std::vector<OutBatch> repack(const ExpandResult &r, size_t batch = BATCH_SIZE) {
    std::vector<OutBatch> out;
    for (size_t i = 0; i < r.dest.size(); i += batch) {
        const size_t e = std::min(r.dest.size(), i + batch);
        OutBatch b;
        b.node_ids.assign(r.dest.begin() + i, r.dest.begin() + e);
        b.selection.reserve(e - i);
        for (size_t k = i; k < e; k++) {
            if (r.row_idx[k] >= BATCH_SIZE) throw std::runtime_error("repack: parent row outside a BATCH_SIZE input batch");
            b.selection.push_back((uint16_t)r.row_idx[k]);
        }
        out.push_back(std::move(b));
    }
    return out;
}

} // namespace fdb
