// shortest_path.hpp -- the shortestPath((a)-[:R1|R2*min..max]->(b)) expression (graph/src/runtime/eval.rs:1296-1513) over live
// relationship tensors.  The reference runs a bidirectional BFS per row over versioned row iterators (NeighborIter, eval.rs:129-244)
// and looks up one relationship per consecutive pair (get_src_dest_relationships(from, to).next(), else (to, from)).
// shortest_path does the same in two library calls for a whole batch: B200_shortest_path over each side's layers, then one
// B200_expand_edges(DIR_BOTH, targets, EDGES_FIRST) over every consecutive pair, whose first entry per row is exactly "forward
// lookup, else reverse".  shortest_path_by_iter restates eval.rs statement for statement, for tests and measurement.
#pragma once
#include "cond_traverse.hpp"
#include <unordered_map>

namespace fdb {

// `adj`: the graph's adjacency VersionedMatrix, walked when no type is named.  `all_types`: every relationship type's Tensor in schema
// order.  `named`: the pattern's types, a null entry for a type the graph lacks (dropped, as the reference's filter_map does).
// max_hops UINT64_MAX: unbounded.  min_hops is 0 or 1 (the parser rejects anything else).
struct ShortestPathQuery {
    const VersionedMatrix *adj = nullptr;
    std::vector<const Tensor *> all_types, named;
    bool directed = true;
    uint64_t min_hops = 1, max_hops = UINT64_MAX;
    std::vector<uint64_t> srcs, dsts;
};

// row i: found[i]; its nodes p[i] .. p[i+1] from src to dst; its relationship ids ep[i] .. ep[i+1] (an id is omitted where neither
// direction holds one)
struct ShortestPathResult {
    std::vector<uint8_t> found;
    std::vector<uint64_t> p{0}, nodes, ep{0}, ids;
};

inline std::vector<const Tensor *> sp_present(const ShortestPathQuery &q) {
    std::vector<const Tensor *> ts;
    for (const Tensor *t : q.named) if (t) ts.push_back(t);
    return ts;
}
// get_src_dest_relationships' types: the named ones the graph has, or every type when none is named
inline std::vector<const Tensor *> sp_edge_types(const ShortestPathQuery &q) { return q.named.empty() ? q.all_types : sp_present(q); }

// the rows found per pair (nodes), then ids by get_edge(from, to, &id) for every consecutive pair
template <class GetIds>
inline ShortestPathResult sp_collect(const std::vector<std::vector<uint64_t>> &paths, const std::vector<uint8_t> &found, GetIds get_ids) {
    ShortestPathResult r;
    r.found = found;
    std::vector<uint64_t> from, to;
    for (const std::vector<uint64_t> &path : paths) {
        r.nodes.insert(r.nodes.end(), path.begin(), path.end());
        r.p.push_back(r.nodes.size());
        for (size_t k = 0; k + 1 < path.size(); k++) { from.push_back(path[k]); to.push_back(path[k + 1]); }
    }
    std::vector<uint8_t> has(from.size(), 0);
    std::vector<uint64_t> id(from.size(), 0);
    if (!from.empty()) get_ids(from, to, has, id);
    size_t e = 0;
    for (const std::vector<uint64_t> &path : paths) {
        for (size_t k = 0; k + 1 < path.size(); k++, e++) if (has[e]) r.ids.push_back(id[e]);
        r.ep.push_back(r.ids.size());
    }
    return r;
}

// rows with src == dst, or with no neighbour on either side: the zero-hop path (min_hops == 0, src == dst) or Null
inline std::vector<uint64_t> sp_trivial(const ShortestPathQuery &q, size_t i, bool *found) {
    *found = q.min_hops == 0 && q.srcs[i] == q.dsts[i];
    return *found ? std::vector<uint64_t>{q.srcs[i]} : std::vector<uint64_t>{};
}

// the library route: one B200_shortest_path call, then one B200_expand_edges call for every consecutive pair
inline ShortestPathResult shortest_path(const ShortestPathQuery &q) {
    if (q.srcs.size() != q.dsts.size()) throw std::invalid_argument("shortest_path: one dst per src");
    const size_t np = q.srcs.size();
    // the sides (NeighborIter::new / new_reversed): typed, forward layers of each type (and matrix_t when undirected); untyped, the
    // adjacency (and every matrix_t when undirected); the backward side of a directed pattern, matrix_t of each type
    std::vector<GrB_Matrix> fm, fdp, fdm, bm, bdp, bdm;
    auto add_vm = [](const VersionedMatrix &v, std::vector<GrB_Matrix> &m, std::vector<GrB_Matrix> &dp, std::vector<GrB_Matrix> &dm) {
        v.wait_all();
        m.push_back(v.m().inner()); dp.push_back(v.dp().inner()); dm.push_back(v.dm().inner());
    };
    const std::vector<const Tensor *> types = q.named.empty() ? q.all_types : sp_present(q);
    if (q.named.empty() && q.adj) add_vm(*q.adj, fm, fdp, fdm);
    for (const Tensor *t : q.named.empty() ? std::vector<const Tensor *>{} : types) {
        t->wait_fwd();
        t->fwd_m().wait(); t->fwd_dp().wait(); t->fwd_dm().wait();
        fm.push_back(t->fwd_m().inner()); fdp.push_back(t->fwd_dp().inner()); fdm.push_back(t->fwd_dm().inner());
    }
    for (const Tensor *t : types) add_vm(t->matrix_t(), q.directed ? bm : fm, q.directed ? bdp : fdp, q.directed ? bdm : fdm);
    if (!q.directed) { bm = fm; bdp = fdp; bdm = fdm; }
    std::vector<std::vector<uint64_t>> paths(np);
    std::vector<uint8_t> found(np, 0);
    if (fm.empty() && bm.empty()) {                  // no relationship to walk: every row is trivial
        for (size_t i = 0; i < np; i++) { bool f; paths[i] = sp_trivial(q, i, &f); found[i] = f; }
        return sp_collect(paths, found, [](auto &, auto &, auto &, auto &) {});
    }
    // one side without an operand (a directed pattern over an adjacency and no relationship type) walks an empty matrix: its
    // front never grows, as NeighborIter::new_reversed over no matrix_t, but the other side can still meet its endpoint
    GrB_Index nv = 0;
    grb_ok(GrB_Matrix_ncols(&nv, fm.empty() ? bm[0] : fm[0]), "GrB_Matrix_ncols");
    Matrix<bool> none(nv, nv);
    for (auto *side : {&fm, &bm})
        if (side->empty()) side->push_back(none.inner());
    if (fdp.size() < fm.size()) { fdp.push_back(nullptr); fdm.push_back(nullptr); }
    if (bdp.size() < bm.size()) { bdp.push_back(nullptr); bdm.push_back(nullptr); }
    std::vector<uint64_t> p(np + 1);
    // a path has at most max_hops + 1 nodes: with a bound up to 31 the first guess always fits, so the BFS runs once
    std::vector<uint32_t> nodes(std::max<size_t>(1024, np * (size_t)std::min<uint64_t>(q.max_hops, 31) + np));
    uint64_t nn = 0;
    for (int attempt = 0; attempt < 2; attempt++) {  // a result larger than the first guess is rerun into its size
        GrB_Info info = B200_shortest_path(q.srcs.data(), q.dsts.data(), np, fm.data(), fdp.data(), fdm.data(), (int)fm.size(), bm.data(),
                                           bdp.data(), bdm.data(), (int)bm.size(), q.min_hops, q.max_hops, p.data(), nodes.data(),
                                           nodes.size(), &nn);
        if (info == GrB_INSUFFICIENT_SPACE && attempt == 0) { nodes.resize(nn); continue; }
        grb_ok(info, "B200_shortest_path");
        break;
    }
    for (size_t i = 0; i < np; i++) {
        paths[i].assign(nodes.begin() + p[i], nodes.begin() + p[i + 1]);
        found[i] = p[i + 1] > p[i];
    }
    const std::vector<const Tensor *> et = sp_edge_types(q);
    return sp_collect(paths, found, [&](const std::vector<uint64_t> &from, const std::vector<uint64_t> &to, std::vector<uint8_t> &has,
                                        std::vector<uint64_t> &id) {
        if (et.empty()) return;
        EdgeExpansion e = expand_edges(from, &to, et, B200_DIR_BOTH, B200_EDGES_FIRST);
        for (size_t k = 0; k < from.size(); k++) if (e.p[k + 1] > e.p[k]) { has[k] = 1; id[k] = e.edge[e.p[k]]; }
    });
}

// ---- the reference's route, statement for statement ----
// NeighborIter (eval.rs:140-244): row iterators over versioned layers, seeked per node; sorted and deduplicated when several
class SpNeighborIter {
    std::vector<LayerIter<uint64_t>> tfwd;               // typed forward layers (structural_iter)
    std::vector<VersionedMatrix::Iter> vfwd, bwd;        // the adjacency, and matrix_t of types
    bool dedup = false;
    std::vector<uint64_t> buf;
  public:
    SpNeighborIter(const ShortestPathQuery &q, bool reversed) {
        const std::vector<const Tensor *> types = q.named.empty() ? q.all_types : sp_present(q);
        if (reversed) {                                  // new_reversed: matrix_t of each type
            for (const Tensor *t : types) vfwd.push_back(t->matrix_t().iter(0, 0));
            dedup = vfwd.size() > 1;
            return;
        }
        if (q.named.empty()) {
            if (q.adj) vfwd.push_back(q.adj->iter(0, 0));
        } else {
            for (const Tensor *t : types) tfwd.push_back(t->fwd_iter(0, 0));
        }
        if (!q.directed)
            for (const Tensor *t : types) bwd.push_back(t->matrix_t().iter(0, 0));
        dedup = tfwd.size() + vfwd.size() + bwd.size() > 1;
    }
    const std::vector<uint64_t> &neighbors(uint64_t node) {
        buf.clear();
        for (auto &it : tfwd) { it.seek(node, node); std::tuple<uint64_t, uint64_t, uint64_t> t; while (it.next(t)) buf.push_back(std::get<1>(t)); }
        for (auto *its : {&vfwd, &bwd})
            for (auto &it : *its) { it.seek(node, node); std::tuple<uint64_t, uint64_t> t; while (it.next(t)) buf.push_back(std::get<1>(t)); }
        if (dedup) { std::sort(buf.begin(), buf.end()); buf.erase(std::unique(buf.begin(), buf.end()), buf.end()); }
        return buf;
    }
};

// bfs_shortest_path (eval.rs:1386-1488): the node list, empty for Null
inline std::vector<uint64_t> sp_bfs_by_iter(SpNeighborIter &fwd_nbrs, SpNeighborIter &bwd_nbrs, uint64_t src, uint64_t dst,
                                            uint64_t max_level, uint64_t min_hops) {
    if (src == dst) return {};
    std::unordered_map<uint64_t, std::pair<uint64_t, uint64_t>> f_map, b_map;   // node -> (parent, depth)
    f_map[src] = {src, 0};
    b_map[dst] = {dst, 0};
    std::vector<uint64_t> f_front{src}, b_front{dst}, next;
    uint64_t df = 0, db = 0;
    bool have_meet = false;
    uint64_t best_od = 0, meet_node = 0;
    while (!have_meet) {
        if (f_front.empty() || b_front.empty() || df + db >= max_level) return {};
        const bool expand_fwd = f_front.size() <= b_front.size();
        std::vector<uint64_t> &front = expand_fwd ? f_front : b_front;
        auto &own = expand_fwd ? f_map : b_map;
        auto &other = expand_fwd ? b_map : f_map;
        SpNeighborIter &nbrs = expand_fwd ? fwd_nbrs : bwd_nbrs;
        const uint64_t depth = (expand_fwd ? df : db) + 1;
        next.clear();
        for (uint64_t cur : front) {
            for (uint64_t nb : nbrs.neighbors(cur)) {
                if (own.count(nb)) continue;
                own[nb] = {cur, depth};
                auto o = other.find(nb);
                if (o != other.end()) {
                    const uint64_t od = o->second.second;
                    if (!have_meet || od < best_od) { have_meet = true; best_od = od; meet_node = nb; }
                } else {
                    next.push_back(nb);
                }
            }
        }
        std::swap(front, next);
        if (expand_fwd) df = depth; else db = depth;
    }
    std::vector<uint64_t> path{meet_node};
    uint64_t cur = meet_node;
    while (cur != src) { cur = f_map.at(cur).first; path.push_back(cur); }
    std::reverse(path.begin(), path.end());
    cur = meet_node;
    while (cur != dst) { cur = b_map.at(cur).first; path.push_back(cur); }
    if (path.size() - 1 < min_hops) return {};
    return path;
}

inline ShortestPathResult shortest_path_by_iter(const ShortestPathQuery &q) {
    if (q.srcs.size() != q.dsts.size()) throw std::invalid_argument("shortest_path: one dst per src");
    const size_t np = q.srcs.size();
    std::vector<std::vector<uint64_t>> paths(np);
    std::vector<uint8_t> found(np, 0);
    for (size_t i = 0; i < np; i++) {                // eval_shortest_path, one row at a time
        if (q.min_hops == 0 && q.srcs[i] == q.dsts[i]) { paths[i] = {q.srcs[i]}; found[i] = 1; continue; }
        SpNeighborIter fwd(q, false), bwd(q, q.directed);
        paths[i] = sp_bfs_by_iter(fwd, bwd, q.srcs[i], q.dsts[i], q.max_hops, q.min_hops);
        found[i] = !paths[i].empty();
    }
    const std::vector<const Tensor *> et = sp_edge_types(q);
    return sp_collect(paths, found, [&](const std::vector<uint64_t> &from, const std::vector<uint64_t> &to, std::vector<uint8_t> &has,
                                        std::vector<uint64_t> &id) {
        for (size_t k = 0; k < from.size(); k++)
            for (int rev = 0; rev < 2 && !has[k]; rev++)
                for (const Tensor *t : et) {
                    std::vector<uint64_t> ids = rev ? t->get(to[k], from[k]) : t->get(from[k], to[k]);
                    if (!ids.empty()) { has[k] = 1; id[k] = ids[0]; break; }
                }
    });
}

} // namespace fdb
