// all_shortest_paths.hpp -- allShortestPaths((a)-[:R1|R2*..k]->(b)) (AllShortestPathsOp::expand_row,
// graph/src/runtime/ops/all_shortest_paths.rs:82-302) over live relationship tensors.  The reference runs, per row, a FIFO BFS
// from src over Graph::get_node_relationships_by_type (one versioned row-iterator seek per type and direction per visited node)
// with hash-map predecessor lists, then a DFS from dst that emits every shortest path.
// all_shortest_paths does the same for a whole batch in B200_all_shortest_paths calls: one that counts, then fills in windows
// (the reference's emitter drains a row across output batches the same way).  all_shortest_paths_by_iter restates expand_row
// statement for statement over TypesAdjacency, for tests and measurement.  Edge-attribute filters are not mirrored: an operator
// with one keeps the reference route.
#pragma once
#include "cond_var_len_traverse.hpp"
#include <deque>
#include <unordered_map>

namespace fdb {

// `all_types`: every relationship type's Tensor in schema order.  `named`: the pattern's types, a null entry for a type the graph
// lacks (dropped); none named: every type (not the adjacency matrix).  directed: Outgoing, else Both.  max_hops UINT64_MAX:
// unbounded; min_hops is 1 (the planner rejects anything else).
struct AllShortestPathsQuery {
    std::vector<const Tensor *> all_types, named;
    bool directed = true;
    uint64_t max_hops = UINT64_MAX;
    std::vector<uint64_t> srcs, dsts;
};

// pair i: count[i] paths of len[i] edges, its paths pp[i] .. pp[i+1]; path k's edges at edges[E_k .. E_k + len), its nodes at
// nodes[E_k + k .. E_k + k + len] (E_k: the edges of the paths before it), as B200_all_shortest_paths lays them out
struct AllShortestPathsResult {
    std::vector<uint64_t> pp{0}, count, len, edges, nodes;
};

inline std::vector<const Tensor *> asp_types(const AllShortestPathsQuery &q) {
    if (q.named.empty()) return q.all_types;
    std::vector<const Tensor *> ts;
    for (const Tensor *t : q.named) if (t) ts.push_back(t);
    return ts;
}

// the library route: one counting call, then calls that fill windows of at most `window` edges until every pair is drained
inline AllShortestPathsResult all_shortest_paths(const AllShortestPathsQuery &q, uint64_t window = (uint64_t)1 << 22) {
    if (q.srcs.size() != q.dsts.size()) throw std::invalid_argument("all_shortest_paths: one dst per src");
    const size_t np = q.srcs.size();
    AllShortestPathsResult r;
    r.pp.assign(np + 1, 0); r.count.assign(np, 0); r.len.assign(np, 0);
    const std::vector<const Tensor *> types = asp_types(q);
    if (types.empty() || np == 0) return r;          // no relationship to walk: no path
    std::vector<B200_TensorLayers> ls;
    for (const Tensor *t : types) ls.push_back(t->waited_layers());
    const int dir = q.directed ? B200_DIR_OUT : B200_DIR_BOTH;
    std::vector<uint64_t> first(np, 0), out_p(np + 1, 0);
    std::vector<uint32_t> len(np, 0);
    uint64_t ne = 0, maxlen = 0, total = 0;
    auto call = [&](uint64_t *pe, uint32_t *pn, uint64_t cap) {
        grb_ok(B200_all_shortest_paths(q.srcs.data(), q.dsts.data(), np, ls.data(), (int)ls.size(), dir, q.max_hops, first.data(),
                                       r.count.data(), len.data(), out_p.data(), pe, pn, cap, &ne), "B200_all_shortest_paths");
    };
    call(nullptr, nullptr, 0);
    for (size_t i = 0; i < np; i++) {
        r.len[i] = len[i];
        maxlen = std::max<uint64_t>(maxlen, len[i]);
        if (r.count[i] > ((uint64_t)1 << 40) - total) throw std::length_error("all_shortest_paths: too many paths to list");
        total += r.count[i];
    }
    std::vector<std::vector<uint64_t>> pe(np), pn(np);
    const uint64_t cap = std::max<uint64_t>(window, maxlen);
    std::vector<uint64_t> eb(cap);
    std::vector<uint32_t> nb(2 * cap);
    for (size_t i0 = 0; i0 < np;) {                  // pairs before i0 are drained
        call(eb.data(), nb.data(), cap);
        uint64_t e = 0;
        for (size_t i = 0; i < np; i++) {
            const uint64_t w = out_p[i + 1] - out_p[i];
            pe[i].insert(pe[i].end(), eb.begin() + e, eb.begin() + e + w * len[i]);
            pn[i].insert(pn[i].end(), nb.begin() + e + out_p[i], nb.begin() + e + out_p[i] + w * (len[i] + 1));
            e += w * len[i];
            first[i] += w;
        }
        while (i0 < np && first[i0] >= r.count[i0]) i0++;
    }
    for (size_t i = 0; i < np; i++) {
        r.edges.insert(r.edges.end(), pe[i].begin(), pe[i].end());
        r.nodes.insert(r.nodes.end(), pn[i].begin(), pn[i].end());
        r.pp[i + 1] = r.pp[i] + r.count[i];
    }
    return r;
}

// ---- the reference's route, statement for statement ----
// expand_row (:128-302) for one pair: the paths in emission order, each as (edges, nodes)
inline void asp_expand_row(const TypesAdjacency &adj, bool bidirectional, uint64_t max_hops, uint64_t src, uint64_t dst,
                           std::vector<std::pair<std::vector<uint64_t>, std::vector<uint64_t>>> &out) {
    std::unordered_map<uint64_t, std::vector<std::pair<uint64_t, uint64_t>>> predecessors;   // node -> (prev, edge id)
    std::unordered_map<uint64_t, uint64_t> distances;
    std::deque<uint64_t> queue;
    const bool is_cycle = src == dst;
    distances[src] = 0;
    queue.push_back(src);
    bool have_sd = false;
    uint64_t sd = 0;
    const EdgeDirection dir = bidirectional ? EdgeDirection::Both : EdgeDirection::Outgoing;
    while (!queue.empty()) {
        const uint64_t current = queue.front();
        queue.pop_front();
        const uint64_t d = distances[current];
        if (have_sd && d >= sd) continue;
        if (d >= max_hops) continue;
        for (const Edge &e : adj(current, dir)) {
            uint64_t next;
            if (e.src == current) next = e.dst;
            else if (bidirectional && e.dst == current) next = e.src;
            else continue;
            const uint64_t nd = d + 1;
            if (is_cycle && next == src) {           // min_hops is 1, so every closing edge counts
                if (!have_sd) { have_sd = true; sd = nd; predecessors[next].push_back({current, e.id}); }
                else if (nd == sd) predecessors[next].push_back({current, e.id});
                continue;
            }
            auto it = distances.find(next);
            if (it != distances.end()) {
                if (nd == it->second) predecessors[next].push_back({current, e.id});
            } else {
                distances[next] = nd;
                predecessors[next].push_back({current, e.id});
                if (next == dst) { have_sd = true; sd = nd; }
                if (nd < max_hops) queue.push_back(next);
            }
        }
    }
    if (!predecessors.count(dst)) return;
    struct State { uint64_t node; std::vector<uint64_t> edges, nodes; };
    std::vector<State> stack{{dst, {}, {dst}}};
    while (!stack.empty()) {
        State st = std::move(stack.back());
        stack.pop_back();
        if (st.node == src && !st.edges.empty()) {
            if (!is_cycle) { std::reverse(st.edges.begin(), st.edges.end()); std::reverse(st.nodes.begin(), st.nodes.end()); }
            out.push_back({std::move(st.edges), std::move(st.nodes)});
            continue;
        }
        auto p = predecessors.find(st.node);
        if (p == predecessors.end()) continue;
        for (const auto &pr : p->second) {
            State n{pr.first, st.edges, st.nodes};
            n.edges.push_back(pr.second);
            n.nodes.push_back(pr.first);
            stack.push_back(std::move(n));
        }
    }
}

inline AllShortestPathsResult all_shortest_paths_by_iter(const AllShortestPathsQuery &q) {
    if (q.srcs.size() != q.dsts.size()) throw std::invalid_argument("all_shortest_paths: one dst per src");
    const std::vector<const Tensor *> types = asp_types(q);
    for (const Tensor *t : types) t->wait();
    TypesAdjacency adj;
    for (const Tensor *t : types) adj.ts.push_back(TensorAdjacency{t});
    AllShortestPathsResult r;
    for (size_t i = 0; i < q.srcs.size(); i++) {     // one row at a time
        std::vector<std::pair<std::vector<uint64_t>, std::vector<uint64_t>>> paths;
        asp_expand_row(adj, !q.directed, q.max_hops, q.srcs[i], q.dsts[i], paths);
        for (auto &p : paths) {
            r.edges.insert(r.edges.end(), p.first.begin(), p.first.end());
            r.nodes.insert(r.nodes.end(), p.second.begin(), p.second.end());
        }
        r.count.push_back(paths.size());
        r.len.push_back(paths.empty() ? 0 : paths[0].first.size());
        r.pp.push_back(r.pp.back() + paths.size());
    }
    return r;
}

} // namespace fdb
