// algo_procs.hpp -- the algo.pageRank, algo.WCC and algo.labelPropagation procedures (graph/src/runtime/functions/
// algo_procedures.rs:687-880, 1168-1270) over live relationship tensors.  The reference builds the adjacency afresh on every call:
// unfiltered, build_adjacency_matrix / build_symmetric_adjacency_matrix (graph.rs:3870-3907) + dup + resize to node_count +
// deleted_nodes_count; with a label filter, a host walk over every edge of the tensors remapped through a hash map
// (build_compact_adj_*_from_tensors, :535-670).  algo_procs builds it in one library call, B200_adjacency_delta over the matrices'
// (m, dp, dm) layers as they stand, then runs the same LAGraph call and output loop.
#pragma once
#include "cond_traverse.hpp"
#include <algorithm>
#include <unordered_map>

namespace fdb {

enum class AlgoProc { PageRank, WCC, CDLP };

// `adj`: the graph's adjacency VersionedMatrix (unfiltered, no type named).  `all_types`: every relationship type's Tensor (compact,
// no type named).  `named` / `labels`: what the call names; a null entry is a name the graph does not have (it contributes nothing).
// pageRank names at most one label.  `node_count`: live nodes; `deleted`: the deleted node ids, so node ids run below node_count +
// deleted.size().
struct AlgoQuery {
    AlgoProc proc = AlgoProc::PageRank;
    const VersionedMatrix *adj = nullptr;
    std::vector<const Tensor *> all_types, named;
    std::vector<const VersionedMatrix *> labels;
    uint64_t node_count = 0;
    std::vector<uint64_t> deleted;
    int max_iterations = 10;                     // CDLP's maxIterations (:1184-1193)
};

// one row per node the procedure returns: pageRank's score, or WCC's componentId / CDLP's communityId (a compact index, returned
// unmapped as the reference does, :859-867, 1249-1257)
struct AlgoResult {
    std::vector<uint64_t> nodes;
    std::vector<double> score;
    std::vector<int64_t> id;
};

// what both routes build: the filter decision and, compact, the kept ids (collect_node_ids' union of the labels' diagonals, :456-477)
struct AlgoPlan {
    bool empty = false;                          // the procedure returns no rows without running
    bool compact = false;
    bool symmetric = false;
    uint64_t n_out = 0;                          // unfiltered: node_count + deleted_nodes_count
    std::vector<uint64_t> keep;                  // compact: ascending node ids, compact index = position
};

inline AlgoPlan algo_plan(const AlgoQuery &q) {
    AlgoPlan p;
    p.symmetric = q.proc != AlgoProc::PageRank;
    p.n_out = q.node_count + q.deleted.size();
    if (q.node_count == 0) { p.empty = true; return p; }
    if (q.labels.empty()) return p;
    if (q.proc == AlgoProc::PageRank) {          // a label covering every node runs unfiltered (:714-716)
        if (q.labels.size() != 1) throw std::invalid_argument("algo.pageRank takes one label");
        if ((q.labels[0] ? q.labels[0]->nvals() : 0) == q.node_count) return p;
    }
    p.compact = true;
    for (const VersionedMatrix *l : q.labels) {
        if (!l) continue;
        auto it = l->iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) if (std::get<0>(t) == std::get<1>(t)) p.keep.push_back(std::get<0>(t));
    }
    std::sort(p.keep.begin(), p.keep.end());
    p.keep.erase(std::unique(p.keep.begin(), p.keep.end()), p.keep.end());
    if (p.keep.empty() && q.proc != AlgoProc::PageRank) p.empty = true;   // WCC / CDLP: an empty node set returns nothing (:826, 1217)
    return p;
}

// the tensors a compact build walks: the named ones that exist, or every type when none is named (:566-577)
inline std::vector<const Tensor *> algo_types(const AlgoQuery &q) {
    std::vector<const Tensor *> out;
    for (const Tensor *t : q.named.empty() ? q.all_types : q.named) if (t) out.push_back(t);
    return out;
}

// LAGraph on the built matrix (which the graph takes over), then the output loop: deleted nodes skipped, compact indices mapped
// back to node ids
inline AlgoResult algo_run(const AlgoQuery &q, const AlgoPlan &p, GrB_Matrix A) {
    GrB_Index n = 0;
    grb_ok(GrB_Matrix_nrows(&n, A), "GrB_Matrix_nrows");
    LAGraph_Graph G = nullptr;
    const bool directed = q.proc == AlgoProc::PageRank;
    int info = LAGraph_New(&G, &A, directed ? LAGraph_ADJACENCY_DIRECTED : LAGraph_ADJACENCY_UNDIRECTED, nullptr);
    if (info) { GrB_Matrix_free(&A); grb_ok((GrB_Info)info, "LAGraph_New"); }
    GrB_Vector v = nullptr;
    int iters = 0;
    if (q.proc == AlgoProc::PageRank) {
        LAGraph_Cached_AT(G, nullptr);
        LAGraph_Cached_OutDegree(G, nullptr);
        info = LAGr_PageRank(&v, &iters, G, 0.85f, 1e-4f, 100, nullptr);
    } else {
        G->is_symmetric_structure = 1;
        info = q.proc == AlgoProc::WCC ? LAGr_ConnectedComponents(&v, G, nullptr) : LAGraph_cdlp(&v, G, q.max_iterations, nullptr);
    }
    LAGraph_Delete(&G, nullptr);
    grb_ok((GrB_Info)info, q.proc == AlgoProc::PageRank ? "LAGr_PageRank" : q.proc == AlgoProc::WCC ? "LAGr_ConnectedComponents" : "LAGraph_cdlp");
    std::vector<GrB_Index> idx(n);
    std::vector<double> f(directed ? n : 0);
    std::vector<int64_t> x(directed ? 0 : n);
    GrB_Index nv = n;
    info = directed ? GrB_Vector_extractTuples_FP64(idx.data(), f.data(), &nv, v) : GrB_Vector_extractTuples_INT64(idx.data(), x.data(), &nv, v);
    GrB_Vector_free(&v);
    grb_ok((GrB_Info)info, "GrB_Vector_extractTuples");
    AlgoResult r;
    for (GrB_Index k = 0; k < nv; k++) {
        const uint64_t id = p.compact ? p.keep[idx[k]] : idx[k];
        if (std::binary_search(q.deleted.begin(), q.deleted.end(), id)) continue;
        r.nodes.push_back(id);
        if (directed) r.score.push_back(f[k]);
        else r.id.push_back(x[k]);
    }
    return r;
}

// the procedure through the library: one B200_adjacency_delta call over the operands as they stand
inline AlgoResult algo_proc(AlgoQuery q) {
    std::sort(q.deleted.begin(), q.deleted.end());
    const AlgoPlan p = algo_plan(q);
    if (p.empty) return AlgoResult();
    std::vector<GrB_Matrix> m, dp, dm;
    if (p.compact || !q.named.empty()) {
        for (const Tensor *t : algo_types(q)) TraversalMatrix(t).operands(m, dp, dm);
    } else {
        if (!q.adj) throw std::invalid_argument("algo_proc: no adjacency matrix");
        TraversalMatrix(q.adj).operands(m, dp, dm);
    }
    const uint64_t rows = p.compact ? p.keep.size() : p.n_out;
    GrB_Matrix A = nullptr;
    // no operand, or an empty kept list (pageRank's label holding no node; a NULL keep would ask for the identity form): nothing
    // to build
    if (m.empty() || (p.compact && p.keep.empty())) grb_ok(GrB_Matrix_new(&A, GrB_BOOL, rows, rows), "GrB_Matrix_new");
    else grb_ok(B200_adjacency_delta(&A, m.data(), dp.data(), dm.data(), (int)m.size(), p.n_out, p.compact ? p.keep.data() : nullptr,
                                     p.keep.size(), p.symmetric ? 1 : 0), "B200_adjacency_delta");
    return algo_run(q, p, A);
}

// The reference's route, statement for statement, for tests and measurement: build_adjacency_matrix (the adjacency's extract, one
// type's extract, or new + one eWiseAdd per type), with symmetric its transpose and an eWiseAdd into a new matrix, then dup +
// resize; or the compact builders' walk over Tensor::iter_edges with a hash map and one GxB_Matrix_build_Scalar.
inline AlgoResult algo_proc_by_extract(AlgoQuery q) {
    std::sort(q.deleted.begin(), q.deleted.end());
    const AlgoPlan p = algo_plan(q);
    if (p.empty) return AlgoResult();
    if (!q.adj) throw std::invalid_argument("algo_proc_by_extract: no adjacency matrix");
    const uint64_t cap = q.adj->ncols();                        // node_cap
    GrB_Matrix A = nullptr;
    if (!p.compact) {
        Matrix<bool> adj;
        if (q.named.empty()) adj = q.adj->extract();
        else if (q.named.size() == 1) adj = q.named[0] ? q.named[0]->extract() : Matrix<bool>(cap, cap);
        else {
            adj = Matrix<bool>(cap, cap);
            for (const Tensor *t : q.named)
                if (t) { Matrix<bool> e = t->extract(); adj.element_wise_add<bool>(nullptr, nullptr, &e); }
        }
        if (p.symmetric) {
            Matrix<bool> at = adj.transpose(), sym(cap, cap);
            sym.element_wise_add<bool>(nullptr, &adj, &at);
            adj = sym;
        }
        adj.wait();
        grb_ok(GrB_Matrix_dup(&A, adj.inner()), "GrB_Matrix_dup");
        GrB_Info info = GrB_Matrix_resize(A, p.n_out, p.n_out);
        if (!info) info = GrB_Matrix_wait(A, GrB_MATERIALIZE);
        if (info) { GrB_Matrix_free(&A); grb_ok(info, "GrB_Matrix_resize"); }
    } else {
        std::unordered_map<uint64_t, uint64_t> id_to_compact(p.keep.size());
        for (size_t k = 0; k < p.keep.size(); k++) id_to_compact.emplace(p.keep[k], k);
        std::vector<uint64_t> ri, ci;
        for (const Tensor *t : algo_types(q))
            for (const auto &e : t->iter_edges()) {
                auto r = id_to_compact.find(std::get<0>(e)), c = id_to_compact.find(std::get<1>(e));
                if (r == id_to_compact.end() || c == id_to_compact.end()) continue;
                ri.push_back(r->second); ci.push_back(c->second);
                if (p.symmetric) { ri.push_back(c->second); ci.push_back(r->second); }
            }
        Matrix<bool> compact(p.keep.size(), p.keep.size());
        compact.build(ri, ci);
        compact.wait();
        grb_ok(GrB_Matrix_dup(&A, compact.inner()), "GrB_Matrix_dup");
    }
    return algo_run(q, p, A);
}

} // namespace fdb
