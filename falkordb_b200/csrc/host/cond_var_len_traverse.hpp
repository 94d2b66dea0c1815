// cond_var_len_traverse.hpp -- C++ mirror of the trail enumerator of the reference's CondVarLenTraverse operator
// (graph/src/runtime/ops/cond_var_len_traverse.rs:152-386): an explicit-stack DFS over relationship-unique paths (trails) of
// min_hops..max_hops edges from one start node, emitting (from, to) per qualifying trail in the reference's order.
//   begin_start_node :152-183   0-hop emission, initial frame
//   advance          :196-386   pop a frame; enumerate its adjacency (cached per node, :241-244) in storage order; skip used
//                               edges (:248-251); direction handling (:253-265); will_emit / will_continue (:319-326); emissions
//                               of one frame come out in adjacency order (:374-377), continuing frames are pushed in adjacency
//                               order and therefore popped in reverse
// What sits on the GraphBLAS boundary is the adjacency fetch: Graph::get_node_relationships_by_type walks the relationship
// tensors with the row iterator (forward rows for outgoing edges, the transpose mirror for incoming ones: tensor.rs:886,
// matrix.rs:1471-1605) -- here Tensor::fwd_iter / matrix_t over the same C calls.  Path materialisation, edge-attribute and
// WHERE filters are runtime code above this layer and are not mirrored.  The multiplicity-insensitive fast path (emit_path off,
// min_hops <= 1) is the reach loop of grb.py: multi_source_reach / the frontier kernels, not this DFS.
#pragma once
#include "tensor.hpp"
#include <functional>
#include <unordered_map>

namespace fdb {

enum class EdgeDirection { Outgoing, Incoming, Both };
struct Edge { uint64_t src, dst, id; };

// Graph::get_node_relationships_by_type for one relationship tensor: outgoing edges of `node` from the forward tensor (ascending
// destination, then ascending edge id), incoming ones through the transpose mirror (ascending source), both for Both.
inline std::vector<Edge> node_relationships(const Tensor &t, uint64_t node, EdgeDirection dir) {
    std::vector<Edge> out;
    if (dir != EdgeDirection::Incoming) {
        auto it = t.fwd_iter(node, node);
        std::tuple<uint64_t, uint64_t, uint64_t> e;
        while (it.next(e))
            for (uint64_t id : t.get(std::get<0>(e), std::get<1>(e))) out.push_back({std::get<0>(e), std::get<1>(e), id});
    }
    if (dir != EdgeDirection::Outgoing) {
        auto it = t.matrix_t().iter(node, node);
        std::tuple<uint64_t, uint64_t> e;
        while (it.next(e)) {
            if (dir == EdgeDirection::Both && std::get<1>(e) == node) continue;      // a self-loop was listed with the outgoing half
            for (uint64_t id : t.get(std::get<1>(e), node)) out.push_back({std::get<1>(e), node, id});
        }
    }
    return out;
}

// edges / nodes: the trail in walk order from the start (nodes includes the start), filled when emit_path is set; hops: its length
struct VarLenResult { uint64_t from, to; std::vector<uint64_t> edges, nodes; uint64_t hops = 0; };

// Adj: callable (node, EdgeDirection) -> std::vector<Edge>, the adjacency fetch (the only part that touches GraphBLAS)
template <class Adj>
class VarLenIterT {
  public:
    VarLenIterT(Adj adj, uint64_t min_hops, uint64_t max_hops, bool reversed = false, bool bidirectional = false,
                int64_t dest_id = -1, bool emit_path = false)
        : fetch_(adj), min_(min_hops), max_(max_hops), reversed_(reversed), bidir_(bidirectional), dest_(dest_id), emit_path_(emit_path) {}

    // the destination labels (:555-563): a trail emits only at a node holding every label; a null entry is a label the graph
    // lacks, and then nothing emits
    void set_dest_labels(std::vector<const VersionedMatrix *> labels) {
        set_dest_label_check([labels](uint64_t v) {
            for (const VersionedMatrix *l : labels) if (!l || !l->get(v, v)) return false;   // node_has_label_id
            return true;
        });
    }
    void set_dest_label_check(std::function<bool(uint64_t)> f) { label_ok_ = std::move(f); }   // (the same over plain sets)
    void set_dest(int64_t dest_id) { dest_ = dest_id; }

    void begin_start_node(uint64_t start) {                       // :152-183
        start_ = start;
        stack_.clear(); buf_.clear();
        if (min_ == 0 && (dest_ < 0 || (uint64_t)dest_ == start) && has_labels(start))
            buf_.push_back({start, start, {}, emit_path_ ? std::vector<uint64_t>{start} : std::vector<uint64_t>(), 0});
        stack_.push_back({start, {}, emit_path_ ? std::vector<uint64_t>{start} : std::vector<uint64_t>(), 0});
    }
    bool next(VarLenResult &out) {                                // Iterator::next :388-
        while (true) {
            if (!buf_.empty()) { out = std::move(buf_.back()); buf_.pop_back(); return true; }
            if (stack_.empty()) return false;
            advance();
        }
    }

  private:
    struct Frame { uint64_t node; std::vector<uint64_t> used, nodes; uint64_t depth; };
    bool has_labels(uint64_t node) const { return !label_ok_ || label_ok_(node); }
    void advance() {                                              // :196-386
        const EdgeDirection dir = bidir_ ? EdgeDirection::Both : reversed_ ? EdgeDirection::Incoming : EdgeDirection::Outgoing;
        while (!stack_.empty()) {
            Frame f = std::move(stack_.back());
            stack_.pop_back();
            const uint64_t hop = f.depth + 1;
            if (hop > max_) continue;
            auto found = adj_.find(f.node);                      // adjacency lists are cached per node (:241-244)
            if (found == adj_.end()) found = adj_.emplace(f.node, fetch_(f.node, dir)).first;
            std::vector<std::pair<uint64_t, uint64_t>> scratch;   // (edge id, neighbour)
            for (const Edge &e : found->second) {
                if (std::find(f.used.begin(), f.used.end(), e.id) != f.used.end()) continue;   // relationship uniqueness
                bool ok = false;
                uint64_t nb = 0;
                if (reversed_) { if (e.dst == f.node) { ok = true; nb = e.src; } }
                else if (e.src == f.node) { ok = true; nb = e.dst; }
                else if (bidir_ && e.dst == f.node) { ok = true; nb = e.src; }
                if (ok) scratch.push_back({e.id, nb});
            }
            for (auto &pr : scratch) {
                const uint64_t dest = pr.second;
                const bool will_emit = hop >= min_ && (dest_ < 0 || (uint64_t)dest_ == dest) && has_labels(dest);
                const bool will_continue = hop < max_;
                if (!will_emit && !will_continue) continue;
                std::vector<uint64_t> used = f.used, nodes = f.nodes;
                used.push_back(pr.first);
                if (emit_path_) nodes.push_back(dest);
                const uint64_t from = reversed_ ? dest : start_, to = reversed_ ? start_ : dest;
                if (will_emit) buf_.push_back({from, to, emit_path_ ? used : std::vector<uint64_t>(), nodes, hop});
                if (will_continue) stack_.push_back({dest, std::move(used), std::move(nodes), hop});
            }
            if (!buf_.empty()) { std::reverse(buf_.begin(), buf_.end()); return; }   // pop() then yields adjacency order (:374-377)
        }
    }
    Adj fetch_;
    uint64_t min_, max_;
    bool reversed_, bidir_;
    int64_t dest_;
    bool emit_path_;
    uint64_t start_ = 0;
    std::vector<Frame> stack_;
    std::vector<VarLenResult> buf_;
    std::unordered_map<uint64_t, std::vector<Edge>> adj_;
    std::function<bool(uint64_t)> label_ok_;
};

struct TensorAdjacency {
    const Tensor *t;
    std::vector<Edge> operator()(uint64_t node, EdgeDirection dir) const { return node_relationships(*t, node, dir); }
};
// Graph::get_node_relationships_by_type over several relationship types (graph.rs:1797-1835): each type's adjacency (One: a
// callable as Adj above), types in the order given
template <class One>
struct TypesAdjacencyT {
    std::vector<One> ts;
    std::vector<Edge> operator()(uint64_t node, EdgeDirection dir) const {
        std::vector<Edge> out;
        for (const One &t : ts) { std::vector<Edge> e = t(node, dir); out.insert(out.end(), e.begin(), e.end()); }
        return out;
    }
};
typedef TypesAdjacencyT<TensorAdjacency> TypesAdjacency;
struct VarLenIter : VarLenIterT<TensorAdjacency> {
    VarLenIter(const Tensor &t, uint64_t min_hops, uint64_t max_hops, bool reversed = false, bool bidirectional = false,
               int64_t dest_id = -1, bool emit_path = false)
        : VarLenIterT<TensorAdjacency>(TensorAdjacency{&t}, min_hops, max_hops, reversed, bidirectional, dest_id, emit_path) {}
};

// The multiplicity-insensitive fast path of CondVarLenTraverse (emit_path off, a consumer that ignores multiplicity): row i of
// the result holds the DISTINCT nodes the trail DFS reaches from starts[i] over every type in `types`, as one
// B200_reach_batch_delta call over the tensors' (m, dp, dm) -- forward layers for Outgoing, the transpose mirror's for Incoming.
// A shortest walk to v != s is a simple path and a shortest closed walk is a simple cycle, so both are trails and the sets agree.
// min_hops = 0 adds the start itself; max_hops = UINT64_MAX is unbounded.  Both directions (s -> u -> s may reuse one edge) and
// min_hops > 1 are refused: such a pattern keeps the DFS (VarLenIter).
inline Matrix<bool> var_len_reach(const std::vector<const Tensor *> &types, EdgeDirection dir, const std::vector<uint64_t> &starts,
                                  uint64_t min_hops, uint64_t max_hops) {
    if (dir == EdgeDirection::Both) throw std::invalid_argument("var_len_reach: a bidirectional pattern is not a reach");
    if (min_hops > 1) throw std::invalid_argument("var_len_reach: min_hops > 1 is not a reach");
    if (types.empty()) throw std::invalid_argument("var_len_reach: no relationship type");
    std::vector<GrB_Matrix> m, dp, dm;
    for (const Tensor *t : types) {
        if (dir == EdgeDirection::Outgoing) {
            t->wait_fwd();
            t->fwd_m().wait(); t->fwd_dp().wait(); t->fwd_dm().wait();
            m.push_back(t->fwd_m().inner()); dp.push_back(t->fwd_dp().inner()); dm.push_back(t->fwd_dm().inner());
        } else {
            const VersionedMatrix &mt = t->matrix_t();
            mt.wait();
            mt.wait_all();
            m.push_back(mt.m().inner()); dp.push_back(mt.dp().inner()); dm.push_back(mt.dm().inner());
        }
    }
    GrB_Matrix raw = nullptr;
    int64_t levels = 0;
    grb_ok(B200_reach_batch_delta(&raw, starts.data(), starts.size(), m.data(), dp.data(), dm.data(), (int)types.size(),
                                  max_hops > (uint64_t)INT64_MAX ? -1 : (int64_t)max_hops, min_hops == 0 ? 1 : 0, &levels),
           "B200_reach_batch_delta");
    return Matrix<bool>::adopt(raw, false);
}

// The same fast path for a bidirectional pattern, as one B200_var_len_reach_both call over every type's live layers: row i holds
// the DISTINCT nodes the trail DFS reaches from starts[i] under Both.  The reach over A u A' is exact for v != s; the start itself
// is decided by the shortest cycle through it, which the call finds.  min_hops > 1 is refused: such a pattern keeps the DFS.
inline Matrix<bool> var_len_reach_both(const std::vector<const Tensor *> &types, const std::vector<uint64_t> &starts, uint64_t min_hops,
                                       uint64_t max_hops) {
    if (min_hops > 1) throw std::invalid_argument("var_len_reach_both: min_hops > 1 is not a reach");
    if (types.empty()) throw std::invalid_argument("var_len_reach_both: no relationship type");
    std::vector<B200_TensorLayers> ls;
    for (const Tensor *t : types) ls.push_back(t->waited_layers());
    GrB_Matrix raw = nullptr;
    grb_ok(B200_var_len_reach_both(&raw, starts.data(), starts.size(), ls.data(), (int)ls.size(), min_hops, max_hops),
           "B200_var_len_reach_both");
    return Matrix<bool>::adopt(raw, false);
}

// The trails of a batch of starts: start i's results are r[p[i] .. p[i+1]).
struct VarLenBatch { std::vector<uint64_t> p{0}; std::vector<VarLenResult> r; };

// The reference's route: one VarLenIterT over TypesAdjacency per start (dests empty or dests[i] < 0: no fixed destination; a
// null label is one the graph lacks).
inline VarLenBatch var_len_trails_dfs(const std::vector<const Tensor *> &types, EdgeDirection dir, const std::vector<uint64_t> &starts,
                                      const std::vector<int64_t> &dests, uint64_t min_hops, uint64_t max_hops,
                                      const std::vector<const VersionedMatrix *> &labels, bool emit_path) {
    for (const Tensor *t : types) t->wait();
    TypesAdjacency adj;
    for (const Tensor *t : types) adj.ts.push_back(TensorAdjacency{t});
    VarLenIterT<TypesAdjacency> it(adj, min_hops, max_hops, dir == EdgeDirection::Incoming, dir == EdgeDirection::Both,
                                   -1, emit_path);
    it.set_dest_labels(labels);
    VarLenBatch b;
    for (size_t i = 0; i < starts.size(); i++) {
        it.set_dest(dests.empty() ? -1 : dests[i]);
        it.begin_start_node(starts[i]);
        VarLenResult r;
        while (it.next(r)) b.r.push_back(std::move(r));
        b.p.push_back(b.r.size());
    }
    return b;
}

// The device route: one B200_var_len_trails call over every type's live layers (as B200_expand_edges takes them) and the labels'
// (m, dp, dm).  Counts first, then the entries into their exact size; (from, to) from the walk's end as :346-350 maps them.
inline VarLenBatch var_len_trails(const std::vector<const Tensor *> &types, EdgeDirection dir, const std::vector<uint64_t> &starts,
                                  const std::vector<int64_t> &dests, uint64_t min_hops, uint64_t max_hops,
                                  const std::vector<const VersionedMatrix *> &labels, bool emit_path,
                                  uint64_t tree_capacity = UINT64_MAX) {
    std::vector<B200_TensorLayers> ls;
    for (const Tensor *t : types) ls.push_back(t->waited_layers());
    std::vector<GrB_Matrix> lm, ldp, ldm;
    for (const VersionedMatrix *l : labels) {
        if (l) { l->wait(); l->wait_all(); }
        lm.push_back(l ? l->m().inner() : nullptr); ldp.push_back(l ? l->dp().inner() : nullptr); ldm.push_back(l ? l->dm().inner() : nullptr);
    }
    const int d = dir == EdgeDirection::Outgoing ? B200_DIR_OUT : dir == EdgeDirection::Incoming ? B200_DIR_IN : B200_DIR_BOTH;
    const size_t n = starts.size();
    VarLenBatch b;
    b.p.assign(n + 1, 0);
    uint64_t nout = 0, npath = 0;
    auto call = [&](uint32_t *end, uint32_t *hops, uint64_t cap, uint64_t *pe, uint32_t *pn, uint64_t pcap) {
        return B200_var_len_trails(starts.data(), dests.empty() ? nullptr : dests.data(), n, ls.data(), (int)ls.size(), d, min_hops,
                                   max_hops, lm.data(), ldp.data(), ldm.data(), (int)lm.size(), tree_capacity, b.p.data(), end, hops,
                                   cap, pe, pn, pcap, &nout, &npath);
    };
    grb_ok(call(nullptr, nullptr, 0, nullptr, nullptr, 0), "B200_var_len_trails");
    std::vector<uint32_t> end(nout + 1), hops(nout + 1), pn(emit_path ? npath + nout + 1 : 0);
    std::vector<uint64_t> pe(emit_path ? npath + 1 : 0);
    grb_ok(call(end.data(), hops.data(), nout, emit_path ? pe.data() : nullptr, emit_path ? pn.data() : nullptr, npath),
           "B200_var_len_trails");
    uint64_t eb = 0;
    size_t i = 0;
    for (uint64_t k = 0; k < nout; k++) {
        while (b.p[i + 1] <= k) i++;
        VarLenResult r;
        const bool rev = dir == EdgeDirection::Incoming;
        r.from = rev ? end[k] : starts[i];
        r.to = rev ? starts[i] : end[k];
        r.hops = hops[k];
        if (emit_path) {
            r.edges.assign(pe.begin() + eb, pe.begin() + eb + hops[k]);
            r.nodes.assign(pn.begin() + eb + k, pn.begin() + eb + k + hops[k] + 1);
        }
        eb += hops[k];
        b.r.push_back(std::move(r));
    }
    return b;
}

} // namespace fdb
