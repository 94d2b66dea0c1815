// algo_bfs.hpp -- the algo.BFS procedure (graph/src/runtime/functions/algo_procedures.rs:1021-1166) over live relationship
// tensors.  The reference builds the adjacency afresh (build_adjacency_matrix, graph.rs:3870-3893), runs
// LAGr_BreadthFirstSearch_Extended on it and, with the edges column, looks up one relationship per reached vertex
// (get_src_dest_relationships, graph.rs:2496-2513).  algo_bfs does the same in two library calls over the matrices as they stand:
// B200_bfs_delta on their (m, dp, dm) layers, then B200_expand_edges for every (parent, child) pair at once.
#pragma once
#include "cond_traverse.hpp"

namespace fdb {

struct BfsResult {
    std::vector<uint64_t> nodes;   // reached vertices but the source, ascending id
    std::vector<uint64_t> edges;   // with want_edges: one relationship from each node's parent to it
};

// `adj`: the graph's adjacency VersionedMatrix, walked when no type is named.  `all_types`: every relationship type's Tensor, whose
// ids the edges come from when no type is named.  `named`: the named types (at most what the procedure's argument names).
// `deleted`: the deleted node ids; pairs whose child or parent is deleted are skipped.  max_depth < 0: unbounded.
struct BfsQuery {
    const VersionedMatrix *adj = nullptr;
    std::vector<const Tensor *> all_types, named;
    std::vector<uint64_t> deleted;
    uint64_t src = 0;
    int64_t max_depth = -1;
    bool want_edges = false;
};

inline void bfs_check_source(const BfsQuery &q) {
    if (std::binary_search(q.deleted.begin(), q.deleted.end(), q.src)) throw std::invalid_argument("Source node not found in graph");
}

// the output loop (algo_procedures.rs:1100-1146): parent[v] >= 0 (or level[v] >= 0 without edges) names a reached v; the source and
// pairs touching a deleted node are skipped.  get_edge(parent, child) -> whether it found an id, written to *id.
template <class GetEdge>
inline BfsResult bfs_collect(const BfsQuery &q, const std::vector<int64_t> &level, const std::vector<int64_t> &parent, GetEdge get_edge) {
    BfsResult r;
    auto deleted = [&](uint64_t v) { return std::binary_search(q.deleted.begin(), q.deleted.end(), v); };
    std::vector<uint64_t> par, child;
    for (uint64_t v = 0; v < level.size(); v++) {
        if (level[v] < 0 || v == q.src) continue;
        if (deleted(v) || (q.want_edges && deleted((uint64_t)parent[v]))) continue;
        r.nodes.push_back(v);
        if (q.want_edges) { par.push_back((uint64_t)parent[v]); child.push_back(v); }
    }
    if (q.want_edges) get_edge(par, child, r.edges);
    return r;
}

// get_src_dest_relationships' types: the named ones, or every type
inline const std::vector<const Tensor *> &bfs_edge_types(const BfsQuery &q) { return q.named.empty() ? q.all_types : q.named; }

// the procedure through the library: one B200_bfs_delta call, then one B200_expand_edges(parents -> children, OUT, FIRST) call
inline BfsResult algo_bfs(BfsQuery q) {
    std::sort(q.deleted.begin(), q.deleted.end());
    bfs_check_source(q);
    std::vector<GrB_Matrix> m, dp, dm;
    if (q.named.empty()) TraversalMatrix(q.adj).operands(m, dp, dm);
    else TraversalMatrix(q.named).operands(m, dp, dm);
    const uint64_t n = q.adj ? q.adj->ncols() : q.named[0]->fwd_m().ncols();
    std::vector<int64_t> level(n), parent(q.want_edges ? n : 0);
    grb_ok(B200_bfs_delta(m.data(), dp.data(), dm.data(), (int)m.size(), q.src, q.max_depth < 0 ? -1 : q.max_depth, -1, level.data(),
                          q.want_edges ? parent.data() : nullptr, B200_LOC_HOST, nullptr), "B200_bfs_delta");
    return bfs_collect(q, level, parent, [&](const std::vector<uint64_t> &par, const std::vector<uint64_t> &child, std::vector<uint64_t> &out) {
        if (par.empty() || bfs_edge_types(q).empty()) return;
        EdgeExpansion e = expand_edges(par, &child, bfs_edge_types(q), B200_DIR_OUT, B200_EDGES_FIRST);
        for (size_t i = 0; i < par.size(); i++) if (e.p[i + 1] > e.p[i]) out.push_back(e.edge[e.p[i]]);
    });
}

// The reference's route, statement for statement: build_adjacency_matrix's fresh matrix (the adjacency's extract, one type's
// extract, or new + one eWiseAdd per type), LAGr_BreadthFirstSearch_Extended on it, then one Tensor::get per pair.  For tests and
// measurement.
inline BfsResult algo_bfs_by_extract(BfsQuery q) {
    std::sort(q.deleted.begin(), q.deleted.end());
    bfs_check_source(q);
    const uint64_t n = q.adj ? q.adj->ncols() : q.named[0]->fwd_m().ncols();
    Matrix<bool> adj = q.named.empty() ? q.adj->extract() : q.named.size() == 1 ? q.named[0]->extract() : Matrix<bool>(n, n);
    if (q.named.size() > 1)
        for (const Tensor *t : q.named) { Matrix<bool> e = t->extract(); adj.element_wise_add<bool>(nullptr, nullptr, &e); }
    adj.wait();
    LAGraph_Graph G = nullptr;
    GrB_Matrix lent = adj.inner();                 // lent to the graph, detached before LAGraph_Delete (the Matrix frees it)
    grb_ok((GrB_Info)LAGraph_New(&G, &lent, LAGraph_ADJACENCY_DIRECTED, nullptr), "LAGraph_New");
    GrB_Vector lv = nullptr, pv = nullptr;
    int info = LAGr_BreadthFirstSearch_Extended(&lv, q.want_edges ? &pv : nullptr, G, q.src, q.max_depth < 0 ? -1 : q.max_depth, -1,
                                                false, nullptr);
    G->A = nullptr;
    LAGraph_Delete(&G, nullptr);
    grb_ok((GrB_Info)info, "LAGr_BreadthFirstSearch_Extended");
    std::vector<int64_t> level(n, -1), parent(q.want_edges ? n : 0, -1);
    auto unpack = [n](GrB_Vector v, std::vector<int64_t> &out) {
        std::vector<GrB_Index> idx(n);
        std::vector<int64_t> val(n);
        GrB_Index nv = n;
        grb_ok(GrB_Vector_extractTuples_INT64(idx.data(), val.data(), &nv, v), "GrB_Vector_extractTuples_INT64");
        for (GrB_Index k = 0; k < nv; k++) out[idx[k]] = val[k];
        GrB_Vector_free(&v);
    };
    if (q.want_edges) { unpack(pv, parent); level = parent; GrB_Vector_free(&lv); }   // parent entries name the reached vertices
    else unpack(lv, level);
    return bfs_collect(q, level, parent, [&](const std::vector<uint64_t> &par, const std::vector<uint64_t> &child, std::vector<uint64_t> &out) {
        for (size_t i = 0; i < par.size(); i++)
            for (const Tensor *t : bfs_edge_types(q)) {
                std::vector<uint64_t> ids = t->get(par[i], child[i]);
                if (!ids.empty()) { out.push_back(ids[0]); break; }
            }
    });
}

} // namespace fdb
