// host_capi.cpp -- flat C entry points over the C++ host mirror (matrix.hpp / versioned_matrix.hpp /
// cond_traverse.hpp) so tests/ can drive it with ctypes, plus transcriptions of the reference's own unit tests
// at this boundary (graph/src/graph/graphblas/versioned_matrix.rs:1278-1523).  Links against libb200grb.so only.
#include "cond_traverse.hpp"
#include "cond_var_len_traverse.hpp"
#include "algo_bfs.hpp"
#include "algo_procs.hpp"
#include "shortest_path.hpp"
#include "all_shortest_paths.hpp"
#include <functional>
#include <map>
#include <set>
#include <cstring>
#include <set>
#include <sstream>

using namespace fdb;

static thread_local std::string g_msg;
#define REQUIRE(cond, text) do { if (!(cond)) { std::ostringstream os; os << "line " << __LINE__ << ": " << text; throw std::runtime_error(os.str()); } } while (0)

typedef std::vector<uint64_t> Ids;

// ---- versioned_matrix.rs:1265-1330 : fold-policy arithmetic (pure host) ----
static uint64_t threshold(uint64_t k, uint64_t tx) { uint64_t target = k * tx; for (uint64_t d = 1;; d++) if (d * d >= target) return d; }
static const uint64_t HUGE_BASE = UINT64_MAX / 4;

static void t_read_path_balance_point_is_flat_in_base_size() {
    REQUIRE(threshold(READ_FOLD_K, 1) == 287, "threshold(READ_FOLD_K,1)");
    for (uint64_t base : {1000000ULL, 10000000ULL, 100000000ULL, (unsigned long long)HUGE_BASE}) {
        REQUIRE(!should_fold_read(286, 1, base), "286 folds at base " << base);
        REQUIRE(should_fold_read(287, 1, base), "287 does not fold at base " << base);
    }
}
static void t_write_path_is_16x_looser_than_read_path() {
    REQUIRE(threshold(WRITE_FOLD_K, 1) == 4528, "write threshold");
    REQUIRE(threshold(WRITE_FOLD_K, 1) / threshold(READ_FOLD_K, 1) == 15, "ratio");
    REQUIRE(!should_fold(4527, 1, HUGE_BASE), "4527");
    REQUIRE(should_fold(4528, 1, HUGE_BASE), "4528");
}
static void t_balance_point_grows_as_sqrt_of_transaction_size() {
    REQUIRE(threshold(READ_FOLD_K, 1) == 287 && threshold(READ_FOLD_K, 100) == 2864, "sqrt growth");
    for (uint64_t tx : {1ULL, 10ULL, 100ULL, 1000ULL}) {
        uint64_t d = threshold(READ_FOLD_K, tx);
        REQUIRE(!should_fold_read(d - 1, tx, HUGE_BASE), "tx " << tx);
        REQUIRE(should_fold_read(d, tx, HUGE_BASE), "tx " << tx);
    }
}
static void t_delta_comparable_to_base_always_folds() {
    REQUIRE(should_fold(512, UINT64_MAX, 1024), "write hatch");
    REQUIRE(should_fold_read(512, UINT64_MAX, 1024), "read hatch");
}
static void t_tiny_deltas_and_read_only_transactions_never_fold() {
    REQUIRE(!should_fold(MIN_FOLD_DELTA - 1, 1, 0) && !should_fold_read(MIN_FOLD_DELTA - 1, 1, 0), "tiny");
    REQUIRE(!should_fold(UINT64_MAX, 0, 1024) && !should_fold_read(UINT64_MAX, 0, 1024), "tx_added == 0");
}

// ---- versioned_matrix.rs:1332-1472 : delta invariants under a deterministic LCG mutation sequence ----
typedef std::set<std::pair<uint64_t, uint64_t>> Model;
static const uint64_t DIM = 512;

static void assert_invariants(const VersionedMatrix &v, const Model &model) {
    v.wait_all();
    {
        auto it = v.dp().iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) {
            REQUIRE(!v.m().get(std::get<0>(t), std::get<1>(t)), "dp n m != 0 at (" << std::get<0>(t) << "," << std::get<1>(t) << ")");
            REQUIRE(!v.dm().get(std::get<0>(t), std::get<1>(t)), "dp n dm != 0");
        }
    }
    {
        auto it = v.dm().iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) REQUIRE(v.m().get(std::get<0>(t), std::get<1>(t)), "dm not subset of m at (" << std::get<0>(t) << "," << std::get<1>(t) << ")");
    }
    REQUIRE(v.nvals() == model.size(), "|m|+|dp|-|dm| = " << v.nvals() << " but the model holds " << model.size());
    Model effective;
    auto it = v.iter();
    std::tuple<uint64_t, uint64_t> t;
    std::pair<uint64_t, uint64_t> prev(0, 0);
    bool first = true;
    while (it.next(t)) {
        std::pair<uint64_t, uint64_t> cur(std::get<0>(t), std::get<1>(t));
        REQUIRE(first || prev < cur, "Iter is not strictly (row,col)-ascending");
        prev = cur; first = false;
        effective.insert(cur);
    }
    REQUIRE(effective == model, "effective state diverged from the model (" << effective.size() << " vs " << model.size() << ")");
}

static uint64_t next_rand(uint64_t &state) {
    state = state * 6364136223846793005ULL + 1442695040888963407ULL;
    return state >> 33;
}

static void t_delta_invariants_hold_across_mutation_sequences() {
    VersionedMatrix v(DIM, DIM);
    Model model;
    uint64_t rng = 0x5eed1234ULL;
    auto key = [](uint64_t r) { return std::make_pair((r % 24) * 7, (r / 24 % 24) * 11); };
    for (int step = 0; step < 4000; step++) {
        switch (next_rand(rng) % 16) {
        case 0: {
            std::vector<std::pair<uint64_t, uint64_t>> batch;
            for (int q = 0; q < 16; q++) batch.push_back(key(next_rand(rng)));
            v.set_all<false>(batch);
            model.insert(batch.begin(), batch.end());
            break;
        }
        case 1: {
            Model batch;
            for (int q = 0; q < 16; q++) batch.insert(key(next_rand(rng)));
            std::vector<uint64_t> rows, cols;
            for (auto &k : batch) { rows.push_back(k.first); cols.push_back(k.second); }
            Matrix<bool> mask(DIM, DIM);
            mask.build(rows, cols);
            mask.wait();
            v.remove_mask(mask);
            for (auto &k : batch) model.erase(k);
            break;
        }
        case 2: v = v.dup(); break;
        case 3: v.wait(); break;
        case 4: v.fold_oversized(); break;
        case 5: case 6: case 7: case 8: {
            auto k = key(next_rand(rng));
            v.remove(k.first, k.second);
            model.erase(k);
            break;
        }
        default: {
            auto k = key(next_rand(rng));
            v.set(k.first, k.second);
            model.insert(k);
        }
        }
        if (step % 37 == 0) assert_invariants(v, model);
    }
    assert_invariants(v, model);
    REQUIRE(v.m().nvals() > 0, "no fold ever happened: the `m` branches of set/remove were never taken");
}

// ---- versioned_matrix.rs:1481-1523 ----
static void t_folded_entry_deleted_and_re_added_stays_out_of_dp() {
    uint64_t filler = 4 * MIN_FOLD_DELTA;
    VersionedMatrix v0(DIM, DIM);
    std::vector<std::pair<uint64_t, uint64_t>> fill;
    for (uint64_t i = 0; i < filler; i++) fill.push_back({i % DIM, (i / DIM + 1) % DIM});
    v0.set_all<false>(fill);
    std::pair<uint64_t, uint64_t> probe(7, 11);
    v0.set(probe.first, probe.second);
    VersionedMatrix v = v0.dup();
    v.set(300, 301);
    v.wait_all();
    REQUIRE(v.m().get(probe.first, probe.second), "the fold did not move the probe into the committed base");
    REQUIRE(!v.dp().get(probe.first, probe.second), "probe still in dp");
    v.remove(probe.first, probe.second);
    v.wait_all();
    REQUIRE(v.dm().get(probe.first, probe.second), "no tombstone");
    REQUIRE(v.m().get(probe.first, probe.second), "base entry vanished");
    REQUIRE(!v.get(probe.first, probe.second), "deleted entry readable");
    v.set(probe.first, probe.second);
    v.wait_all();
    REQUIRE(!v.dm().get(probe.first, probe.second), "tombstone survived the re-add");
    REQUIRE(!v.dp().get(probe.first, probe.second), "re-add duplicated the committed entry into dp");
    REQUIRE(v.get(probe.first, probe.second), "probe unreadable");
    REQUIRE(v.nvals() == filler + 2, "nvals double-counted the re-add: " << v.nvals());
}

// ---- README.md:85-110 MotoGP demo: 3 riders -rides-> 3 teams; BASELINE config 1 (plumbing) ----
static void t_motogp_two_hop() {
    // node ids: riders 0 Rossi, 1 Marquez, 2 Pedrosa ; teams 3 Yamaha, 4 Honda, 5 Ducati (Ducati has no rider)
    uint64_t n = 16384; // initial node capacity, src/graph_core.rs:471
    VersionedMatrix rides(n, n), rider(n, n), team(n, n);
    rides.set_all<true>({{0, 3}, {1, 4}, {2, 4}});
    for (uint64_t i : {0, 1, 2}) rider.set(i, i);
    for (uint64_t i : {3, 4, 5}) team.set(i, i);
    // MATCH (r:Rider)-[:rides]->(t:Team) WHERE t.name = 'Yamaha' RETURN r.name  => "Valentino Rossi"
    ExpandResult one = expand_batch({0, 1, 2}, {TraversalMatrix(&rides)}, {&rider}, {&team});
    std::vector<uint64_t> who;
    for (size_t k = 0; k < one.dest.size(); k++) if (one.dest[k] == 3) who.push_back(one.row_idx[k]);
    REQUIRE(who.size() == 1 && who[0] == 0, "Yamaha's rider is not Valentino Rossi");
    // MATCH (r:Rider)-[:rides]->(t:Team {name:'Ducati'}) RETURN count(r) ... README expects 1 for Yamaha riders
    size_t yamaha = 0;
    for (uint64_t d : one.dest) yamaha += d == 3;
    REQUIRE(yamaha == 1, "count != 1");
    // second hop through the maintained transpose: rider -> team -> team-mates
    VersionedMatrix rides_t = rides.transpose();
    ExpandResult two = expand_batch({0, 1, 2}, {TraversalMatrix(&rides), TraversalMatrix(&rides_t)}, {&rider}, {&rider});
    std::set<std::pair<uint64_t, uint64_t>> got;
    for (size_t k = 0; k < two.dest.size(); k++) got.insert({two.row_idx[k], two.dest[k]});
    std::set<std::pair<uint64_t, uint64_t>> want = {{0, 0}, {1, 1}, {1, 2}, {2, 1}, {2, 2}};
    REQUIRE(got == want, "2-hop team-mates differ");
    // a pending delete is honoured by the dirty-snapshot path (matrix.rs:1342-1400)
    rides.remove(2, 4);
    ExpandResult three = expand_batch({0, 1, 2}, {TraversalMatrix(&rides)}, {}, {});
    REQUIRE(three.dest.size() == 2, "tombstoned edge still traversed");
}

// ---- tensor.rs:1340-1669 : the per-relationship-type edge store ----
// The writes of these tests go through one of the two routes: the reference's (Tensor::set_all_from_slices / remove_all) or the
// device plans' (set_all_from_slices_dev / remove_all_dev); the *_dev test names run the second.
static bool g_write_dev = false;
static void tensor_add(Tensor &t, const std::vector<uint64_t> &s, const std::vector<uint64_t> &d, const std::vector<uint64_t> &i) {
    if (g_write_dev) t.set_all_from_slices_dev(s, d, i);
    else t.set_all_from_slices(s, d, i);
}
static std::vector<std::pair<uint64_t, uint64_t>> tensor_remove(Tensor &t, const std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> &r) {
    return g_write_dev ? t.remove_all_dev(r) : t.remove_all(r);
}
static uint64_t count_sentinels(const Tensor &t, uint64_t pairs) {
    uint64_t s = 0, v;
    for (uint64_t i = 0; i < pairs; i++) if (t.eff_get(i, i + 1, &v) && v == MULTI_EDGE) s++;
    return s;
}
static void t_multi_pairs_after_within_batch_duplicates() {      // tensor.rs:1340-1380
    for (auto cfg : {std::make_pair(64ULL, 2ULL), std::make_pair(1000ULL, 2ULL), std::make_pair(1000ULL, 4ULL)}) {
        uint64_t pairs = cfg.first, dup = cfg.second, n = pairs + 1, next_id = 0;
        Tensor t(n, n);
        std::vector<uint64_t> srcs, dsts, ids;
        for (uint64_t i = 0; i < pairs; i++) for (uint64_t d = 0; d < dup; d++) { srcs.push_back(i); dsts.push_back(i + 1); ids.push_back(next_id++); }
        tensor_add(t, srcs, dsts, ids);
        t.wait_fwd();
        uint64_t sentinels = count_sentinels(t, pairs), derived = t.multi_pairs(), edges = 0;
        for (uint64_t i = 0; i < pairs; i++) edges += t.get(i, i + 1).size();
        REQUIRE(derived == sentinels, "multi_pairs disagrees (within-batch dups): " << derived << " vs " << sentinels);
        REQUIRE(edges == pairs * dup, "lost edges: " << edges);
        REQUIRE(t.edge_count() == edges, "edge_count " << t.edge_count() << " disagrees with a full scan " << edges);
    }
}
static void t_multi_pairs_matches_the_sentinel_count() {         // tensor.rs:1382-1425
    for (auto cfg : {std::make_pair(64ULL, 2ULL), std::make_pair(1000ULL, 3ULL), std::make_pair(2000ULL, 2ULL)}) {
        uint64_t pairs = cfg.first, dup = cfg.second, n = pairs + 1;
        Tensor t(n, n);
        std::vector<uint64_t> srcs, dsts;
        for (uint64_t i = 0; i < pairs; i++) { srcs.push_back(i); dsts.push_back(i + 1); }
        for (uint64_t round = 0; round < dup; round++) {
            std::vector<uint64_t> ids;
            for (uint64_t i = 0; i < pairs; i++) ids.push_back(round * pairs + i);
            tensor_add(t, srcs, dsts, ids);
        }
        t.wait_fwd();
        uint64_t sentinels = count_sentinels(t, pairs), derived = t.multi_pairs(), edges = 0;
        for (uint64_t i = 0; i < pairs; i++) edges += t.get(i, i + 1).size();
        REQUIRE(derived == sentinels && sentinels == pairs, "multi_pairs " << derived << " sentinels " << sentinels);
        REQUIRE(t.edge_count() == edges && edges == pairs * dup, "edge_count " << t.edge_count() << " vs " << edges);
    }
}
static void t_bulk_remove_and_extract_edge_id_zero() {           // tensor.rs:1427-1476
    const uint64_t N = 10000;
    Tensor t0(N + 1, N + 1);
    std::vector<uint64_t> srcs, dsts, ids;
    for (uint64_t i = 0; i < N; i++) { srcs.push_back(i); dsts.push_back(i + 1); ids.push_back(i); }
    tensor_add(t0, srcs, dsts, ids);
    Tensor t = t0.dup();
    t.flush();
    t.fwd_m().wait();
    REQUIRE(t.fwd_m().contains(0, 1), "edge id 0 not folded into base");
    uint64_t v = 77;
    REQUIRE(t.fwd_m().get(0, 1, &v) && v == 0, "edge id 0 changed value in the fold");
    tensor_remove(t, {std::make_tuple(0ULL, 0ULL, 1ULL), std::make_tuple(5ULL, 5ULL, 6ULL)});
    REQUIRE(t.get(0, 1).empty(), "edge id 0 still readable");
    REQUIRE(t.get(5, 6).empty(), "edge id 5 still readable");
    Matrix<bool> ex = t.extract();
    ex.wait();
    REQUIRE(ex.contains(1, 2), "unrelated live pair (1,2) disappeared");
    REQUIRE(!ex.contains(5, 6), "control pair (5,6) not deleted");
    REQUIRE(!ex.contains(0, 1), "deleted pair (0,1) still present in extract: edge id 0 was typecast to false in dm");
}
static void t_deleting_everything_folds_the_tombstones_away() {  // tensor.rs:1503-1530
    const uint64_t N = 10000;
    Tensor t0(N + 1, N + 1);
    std::vector<uint64_t> srcs, dsts, ids;
    for (uint64_t i = 0; i < N; i++) { srcs.push_back(i); dsts.push_back(i + 1); ids.push_back(i); }
    tensor_add(t0, srcs, dsts, ids);
    Tensor t1 = t0.dup();
    t1.flush();
    t1.wait_fwd();
    REQUIRE(t1.fwd_m().nvals() == N, "adds did not fold into the base");
    Tensor t = t1.dup();
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rels;
    for (uint64_t i = 0; i < N; i++) rels.push_back(std::make_tuple(i, i, i + 1));
    tensor_remove(t, rels);
    t.fold_oversized();
    t.wait_fwd();
    REQUIRE(t.fwd_m().nvals() == 0, "base kept its deleted entries");
    REQUIRE(t.fwd_dm().nvals() == 0, "tombstones kept alongside the base");
    REQUIRE(t.get(0, 1).empty(), "deleted edge still readable");
}
static Tensor committed_pairs(uint64_t n) {                      // tensor.rs:1534-1546
    Tensor t(n + 1, n + 1);
    std::vector<uint64_t> srcs, dsts, ids;
    for (uint64_t i = 0; i < n; i++) for (int k = 0; k < 2; k++) { srcs.push_back(i); dsts.push_back(i + 1); ids.push_back(2 * i + k); }
    tensor_add(t, srcs, dsts, ids);
    t.fold_oversized();
    t.wait();
    REQUIRE(t.fwd_m().nvals() == n, "sentinels not folded into the base");
    return t.dup();
}
static void t_batch_demote_leaves_every_survivor_inline() {      // tensor.rs:1548-1571
    const uint64_t N = 512;
    Tensor t = committed_pairs(N);
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rels;
    for (uint64_t i = 0; i < N; i++) rels.push_back(std::make_tuple(2 * i + 1, i, i + 1));
    auto emptied = tensor_remove(t, rels);
    REQUIRE(emptied.empty(), "demoted pairs reported as emptied");
    REQUIRE(t.edge_count() == N, "edge count after demoting every pair: " << t.edge_count());
    REQUIRE(t.multi_pairs() == 0, "a demoted pair still counts as multi");
    REQUIRE(t.edge_versioned().nvals() == 0, "`me` still holds ids of demoted pairs");
    for (uint64_t i = 0; i < N; i++) { auto g = t.get(i, i + 1); REQUIRE(g.size() == 1 && g[0] == 2 * i, "pair " << i << " lost its surviving edge"); }
}
static void t_batch_can_demote_and_then_empty_the_same_pair() {  // tensor.rs:1573-1615
    const uint64_t N = 512;
    Tensor t = committed_pairs(N);
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rels;
    for (uint64_t i = 0; i < N; i++) {
        rels.push_back(std::make_tuple(2 * i + 1, i, i + 1));
        rels.push_back(std::make_tuple(2 * i + 1, i, i + 1));
        rels.push_back(std::make_tuple(7 * N + i, i, i + 1));
        rels.push_back(std::make_tuple(2 * i, i, i + 1));
        rels.push_back(std::make_tuple(2 * i, i, i + 1));
    }
    auto emptied = tensor_remove(t, rels);
    std::sort(emptied.begin(), emptied.end());
    REQUIRE(emptied.size() == N, "every pair should be reported emptied exactly once: " << emptied.size());
    for (uint64_t i = 0; i < N; i++) REQUIRE(emptied[i] == std::make_pair(i, i + 1), "emptied list wrong at " << i);
    REQUIRE(t.edge_count() == 0, "edges left after removing all of them: " << t.edge_count());
    REQUIRE(t.multi_pairs() == 0 && t.edge_versioned().nvals() == 0, "`me` still holds ids");
    t.matrix_t().wait();
    REQUIRE(t.matrix_t().extract().nvals() == 0, "backward adjacency kept the pairs");
    for (uint64_t i = 0; i < N; i++) REQUIRE(t.get(i, i + 1).empty(), "pair " << i << " still readable");
}
static void t_demoting_to_the_committed_value_cancels_to_clean() {  // tensor.rs:1634-1668
    const uint64_t N = 512;
    Tensor t0(N + 1, N + 1);
    std::vector<uint64_t> srcs, dsts, ids;
    for (uint64_t i = 0; i < N; i++) { srcs.push_back(i); dsts.push_back(i + 1); ids.push_back(i + 1); }
    tensor_add(t0, srcs, dsts, ids);
    t0.fold_oversized();
    t0.wait();
    uint64_t v = 0;
    REQUIRE(t0.fwd_m().get(0, 1, &v) && v == 1, "single edge not committed");
    Tensor t = t0.dup();                          // promote in this version (m = 1, dp = M, me = {1, 9}), then remove the new edge
    tensor_add(t, {0}, {1}, {9});
    auto emptied = tensor_remove(t, {std::make_tuple(9ULL, 0ULL, 1ULL)});
    REQUIRE(emptied.empty(), "surviving pair reported as emptied");
    t.wait();
    REQUIRE(t.fwd_dp().nvals() == 0, "dp still shadows m with m's own value");
    REQUIRE(t.fwd_dm().nvals() == 0, "demotion left a tombstone");
    REQUIRE(t.edge_versioned().nvals() == 0, "`me` not emptied by the demotion");
    REQUIRE(t.edge_count() == N, "edge count after promote + demote: " << t.edge_count());
    auto g = t.get(0, 1);
    REQUIRE(g.size() == 1 && g[0] == 1, "committed edge lost");
}
// CondTraverse over a relationship tensor (TraversalMatrix::U64, cond_traverse.rs:83): the u64 edge ids -- including
// id 0 and the MULTI_EDGE sentinel -- are never read by ANY_PAIR; only the pattern matters.
// batch boundary (batch.rs:81, 274-287): <= 1024 rows per output batch, NodeIds + u16 selection vector, order preserved
static void t_repack_output_batches() {
    const uint64_t n = 4096;
    VersionedMatrix star(n, n);
    for (uint64_t j = 1; j <= 2500; j++) star.set(0, j);          // one parent with 2500 destinations
    for (uint64_t j = 10; j < 40; j++) star.set(3, j);            // another with 30
    star.wait();
    ExpandResult r = expand_batch({0, 7, 2, 3}, {TraversalMatrix(&star)}, {}, {});
    REQUIRE(r.dest.size() == 2530, "expand_batch pair count");
    std::vector<OutBatch> b = repack(r);
    REQUIRE(b.size() == 3 && b[0].node_ids.size() == 1024 && b[1].node_ids.size() == 1024 && b[2].node_ids.size() == 482, "batches of <= 1024 rows");
    size_t k = 0;
    for (const OutBatch &ob : b) {
        REQUIRE(ob.node_ids.size() == ob.selection.size(), "one selection entry per row");
        for (size_t t = 0; t < ob.node_ids.size(); t++, k++) {
            REQUIRE(ob.node_ids[t] == r.dest[k] && ob.selection[t] == r.row_idx[k], "order and parent rows preserved");
            REQUIRE(ob.selection[t] == 0 || ob.selection[t] == 3, "parents are input rows 0 and 3");
        }
    }
    REQUIRE(repack(ExpandResult{}).empty(), "nothing in, nothing out");
}

static void t_repack_logic() {                  // host only: the re-pack itself makes no GraphBLAS call
    ExpandResult r;
    for (uint64_t row : {0ULL, 3ULL, 1023ULL})
        for (uint64_t d = 0; d < (row == 3 ? 1500ULL : 700ULL); d++) { r.row_idx.push_back(row); r.dest.push_back(row * 100000 + d); }
    std::vector<OutBatch> b = repack(r);
    REQUIRE(b.size() == 3 && b[0].node_ids.size() == 1024 && b[1].node_ids.size() == 1024 && b[2].node_ids.size() == 2900 - 2048, "2900 pairs -> 1024 + 1024 + 852");
    size_t k = 0;
    for (const OutBatch &ob : b)
        for (size_t t = 0; t < ob.node_ids.size(); t++, k++)
            REQUIRE(ob.node_ids[t] == r.dest[k] && ob.selection[t] == r.row_idx[k], "order and parent rows preserved at pair " << k);
    REQUIRE(k == 2900 && b[0].selection[699] == 0 && b[0].selection[700] == 3 && b[2].selection.back() == 1023, "parents 0, 3 and 1023 (the largest u16 row of a batch)");
    REQUIRE(repack(r, 4096).size() == 1 && repack(ExpandResult{}).empty(), "one batch when it fits; nothing in, nothing out");
    r.row_idx[5] = BATCH_SIZE;                       // a parent row outside any input batch
    bool threw = false;
    try { repack(r); } catch (const std::runtime_error &) { threw = true; }
    REQUIRE(threw, "a parent row >= BATCH_SIZE is an error, not a truncated u16");
}

// CondVarLenTraverse's trail enumerator (cond_var_len_traverse.rs:152-386) against a brute-force enumeration of every trail:
// a small multigraph with a cycle, a multi-edge pair, a self-loop and a dead end; outgoing, incoming and bidirectional expansion,
// min/max hop windows, a fixed destination, and the emission order inside one frame (adjacency order).  Run twice: over a plain
// in-memory adjacency in tensor storage order (host only: the DFS logic) and over a Tensor through the C ABI (row iterators).
static const std::vector<uint64_t> VL_S{0, 0, 1, 2, 2, 3, 1, 4, 0}, VL_D{1, 1, 2, 0, 3, 3, 4, 5, 6}, VL_I{10, 11, 12, 13, 14, 15, 16, 17, 18};
// edges (src, dst, id):  0->1 (10), 0->1 (11) multi-edge, 1->2 (12), 2->0 (13) closes a cycle, 2->3 (14), 3->3 (15) self-loop,
//                        1->4 (16), 4->5 (17), 0->6 (18) dead end
struct PlainAdjacency {       // what node_relationships returns for the same graph: out by (dst, id), in by (src, id)
    std::vector<Edge> operator()(uint64_t node, EdgeDirection dir) const {
        std::vector<Edge> out, in;
        for (size_t e = 0; e < VL_S.size(); e++) {
            if (VL_S[e] == node) out.push_back({VL_S[e], VL_D[e], VL_I[e]});
            if (VL_D[e] == node && !(dir == EdgeDirection::Both && VL_S[e] == node)) in.push_back({VL_S[e], VL_D[e], VL_I[e]});
        }
        std::sort(out.begin(), out.end(), [](const Edge &a, const Edge &b) { return a.dst != b.dst ? a.dst < b.dst : a.id < b.id; });
        std::sort(in.begin(), in.end(), [](const Edge &a, const Edge &b) { return a.src != b.src ? a.src < b.src : a.id < b.id; });
        std::vector<Edge> r;
        if (dir != EdgeDirection::Incoming) r = out;
        if (dir != EdgeDirection::Outgoing) r.insert(r.end(), in.begin(), in.end());
        return r;
    }
};
static std::multiset<std::pair<uint64_t, uint64_t>> vl_brute(uint64_t start, uint64_t lo, uint64_t hi, int mode /*0 out 1 in 2 both*/, int64_t dest) {
    std::multiset<std::pair<uint64_t, uint64_t>> out;
    if (lo == 0 && (dest < 0 || (uint64_t)dest == start)) out.insert({start, start});
    std::function<void(uint64_t, std::set<uint64_t> &, uint64_t)> go = [&](uint64_t cur, std::set<uint64_t> &used, uint64_t depth) {
        if (depth == hi) return;
        for (size_t e = 0; e < VL_S.size(); e++) {
            if (used.count(VL_I[e])) continue;
            uint64_t nb;
            if ((mode == 0 || mode == 2) && VL_S[e] == cur) nb = VL_D[e];
            else if ((mode == 1 || mode == 2) && VL_D[e] == cur) nb = VL_S[e];
            else continue;
            used.insert(VL_I[e]);
            if (depth + 1 >= lo && (dest < 0 || (uint64_t)dest == nb)) out.insert(mode == 1 ? std::make_pair(nb, start) : std::make_pair(start, nb));
            go(nb, used, depth + 1);
            used.erase(VL_I[e]);
        }
    };
    std::set<uint64_t> used;
    go(start, used, 0);
    return out;
}
template <class MakeIter>
static void vl_check(MakeIter make) {
    for (int mode = 0; mode < 3; mode++)
        for (uint64_t start : {0ull, 1ull, 2ull, 3ull, 5ull, 6ull})
            for (auto win : std::vector<std::pair<uint64_t, uint64_t>>{{1, 1}, {1, 3}, {0, 2}, {2, 5}, {3, 3}, {1, 9}})
                for (int64_t dest : {(int64_t)-1, (int64_t)0, (int64_t)3}) {
                    auto it = make(win.first, win.second, mode == 1, mode == 2, dest);
                    it.begin_start_node(start);
                    std::multiset<std::pair<uint64_t, uint64_t>> got;
                    VarLenResult r;
                    while (it.next(r)) {
                        got.insert({r.from, r.to});
                        std::set<uint64_t> uniq(r.edges.begin(), r.edges.end());
                        REQUIRE(uniq.size() == r.edges.size(), "a trail repeats an edge");
                        REQUIRE(r.edges.size() >= win.first && r.edges.size() <= win.second, "trail length outside the hop window");
                    }
                    REQUIRE(got == vl_brute(start, win.first, win.second, mode, dest),
                            "trails differ: mode " << mode << " start " << start << " hops " << win.first << ".." << win.second << " dest " << dest);
                }
    // emission order inside the first frame = adjacency order: (0,1) via edge 10, (0,1) via edge 11, (0,6)
    auto it = make(1, 1, false, false, -1);
    it.begin_start_node(0);
    std::vector<uint64_t> order;
    VarLenResult r;
    while (it.next(r)) order.push_back(r.edges[0]);
    REQUIRE((order == std::vector<uint64_t>{10, 11, 18}), "first-frame emissions must come out in adjacency order");
}
static void t_var_len_trails_logic() {      // host only: no GraphBLAS call
    vl_check([](uint64_t lo, uint64_t hi, bool rev, bool bi, int64_t dest) { return VarLenIterT<PlainAdjacency>(PlainAdjacency(), lo, hi, rev, bi, dest, true); });
}
static void t_var_len_trails() {            // the same over a Tensor: adjacency through the row iterators of the C ABI
    Tensor t(16, 16);
    t.set_all_from_slices(VL_S, VL_D, VL_I);
    t.wait();
    t.rebuild_backward();
    vl_check([&](uint64_t lo, uint64_t hi, bool rev, bool bi, int64_t dest) { return VarLenIter(t, lo, hi, rev, bi, dest, true); });
}

// The same enumerator over several relationship types (TypesAdjacencyT, get_node_relationships_by_type's order) with destination
// labels, against a brute-force enumeration of every trail over the union of the types' edges: parallel edges on one pair in two
// types and inside one type, self-loops, a cycle, Out / In / Both, fixed destinations, and labels present, absent or missing.
// Host only: the per-type adjacency is a plain edge list in tensor storage order.
struct IdListAdjacency {        // one type: out by (dst, id), in by (src, id); under Both a self-loop only in the out half
    std::vector<uint64_t> S, D, I;
    std::vector<Edge> operator()(uint64_t node, EdgeDirection dir) const {
        std::vector<Edge> out, in;
        for (size_t e = 0; e < S.size(); e++) {
            if (S[e] == node) out.push_back({S[e], D[e], I[e]});
            if (D[e] == node && !(dir == EdgeDirection::Both && S[e] == node)) in.push_back({S[e], D[e], I[e]});
        }
        std::sort(out.begin(), out.end(), [](const Edge &a, const Edge &b) { return a.dst != b.dst ? a.dst < b.dst : a.id < b.id; });
        std::sort(in.begin(), in.end(), [](const Edge &a, const Edge &b) { return a.src != b.src ? a.src < b.src : a.id < b.id; });
        std::vector<Edge> r;
        if (dir != EdgeDirection::Incoming) r = out;
        if (dir != EdgeDirection::Outgoing) r.insert(r.end(), in.begin(), in.end());
        return r;
    }
};
static void t_var_len_types_labels_logic() {
    const std::vector<IdListAdjacency> types = {
        {{0, 0, 1, 2, 2, 3}, {1, 1, 2, 0, 3, 3}, {10, 11, 12, 13, 14, 15}},   // a multi-edge pair (0,1), a cycle, a self-loop at 3
        {{0, 1, 3}, {1, 2, 0}, {20, 21, 22}},                                 // (0,1) and (1,2) again in a second type
        {{1, 2}, {1, 4}, {30, 31}}};                                          // a self-loop at 1, a dead end at 4
    std::vector<Edge> all;
    for (const IdListAdjacency &t : types)
        for (size_t e = 0; e < t.S.size(); e++) all.push_back({t.S[e], t.D[e], t.I[e]});
    const std::set<uint64_t> L1{0, 1, 2, 3}, L2{1, 2, 3};
    typedef std::tuple<uint64_t, uint64_t, std::vector<uint64_t>, std::vector<uint64_t>> Row;
    for (int mode = 0; mode < 3; mode++)
        for (int labs = 0; labs < 4; labs++)             // none, {L1}, {L1, L2}, {L1, missing}
            for (uint64_t start : {0ull, 1ull, 2ull, 3ull, 4ull})
                for (auto win : std::vector<std::pair<uint64_t, uint64_t>>{{0, 0}, {1, 1}, {0, 2}, {2, 4}, {1, 9}})
                    for (int64_t dest : {(int64_t)-1, (int64_t)1, (int64_t)3}) {
                        auto ok = [&](uint64_t v) { return labs == 0 || (L1.count(v) && (labs == 1 || (labs == 2 && L2.count(v)))); };
                        std::multiset<Row> want, got;
                        std::function<void(uint64_t, std::vector<uint64_t> &, std::vector<uint64_t> &)> go =
                            [&](uint64_t cur, std::vector<uint64_t> &used, std::vector<uint64_t> &nodes) {
                                const uint64_t depth = used.size();
                                if (depth >= win.first && (dest < 0 || (uint64_t)dest == cur) && ok(cur))
                                    want.insert(Row{mode == 1 ? cur : start, mode == 1 ? start : cur, used, nodes});
                                if (depth == win.second) return;
                                for (const Edge &e : all) {
                                    if (std::find(used.begin(), used.end(), e.id) != used.end()) continue;
                                    std::vector<uint64_t> nbs;
                                    if (mode != 1 && e.src == cur) nbs.push_back(e.dst);
                                    if (mode != 0 && e.dst == cur && !(mode == 2 && e.src == cur)) nbs.push_back(e.src);
                                    for (uint64_t nb : nbs) {
                                        used.push_back(e.id); nodes.push_back(nb);
                                        go(nb, used, nodes);
                                        used.pop_back(); nodes.pop_back();
                                    }
                                }
                            };
                        std::vector<uint64_t> used, nodes{start};
                        go(start, used, nodes);
                        VarLenIterT<TypesAdjacencyT<IdListAdjacency>> it(TypesAdjacencyT<IdListAdjacency>{types}, win.first, win.second,
                                                                         mode == 1, mode == 2, dest, true);
                        it.set_dest_label_check(ok);
                        it.begin_start_node(start);
                        VarLenResult r;
                        while (it.next(r)) got.insert(Row{r.from, r.to, r.edges, r.nodes});
                        REQUIRE(got == want, "trails over types differ: mode " << mode << " labels " << labs << " start " << start
                                << " hops " << win.first << ".." << win.second << " dest " << dest << " (" << got.size() << " vs "
                                << want.size() << ")");
                    }
    // the first frame of start 0, Out, *1..1: type order first (10, 11 in type 0, then 20 in type 1)
    VarLenIterT<TypesAdjacencyT<IdListAdjacency>> it(TypesAdjacencyT<IdListAdjacency>{types}, 1, 1, false, false, -1, true);
    it.begin_start_node(0);
    std::vector<uint64_t> order;
    VarLenResult r;
    while (it.next(r)) order.push_back(r.edges[0]);
    REQUIRE((order == std::vector<uint64_t>{10, 11, 20}), "emissions follow types in order, then neighbour and id");
}

// The reference's query-level goldens for variable-length traversals (tests/flow/test_variable_length_traversals.py), transcribed
// at the level this mirror covers: which (from, to) pairs and path lengths the trail enumerator yields.  Host only.
struct ListAdjacency {          // node_relationships over explicit edge lists (ids = positions): out by (dst, id), in by (src, id)
    std::vector<uint64_t> S, D;
    std::vector<Edge> operator()(uint64_t node, EdgeDirection dir) const {
        std::vector<Edge> out, in;
        for (size_t e = 0; e < S.size(); e++) {
            if (S[e] == node) out.push_back({S[e], D[e], (uint64_t)e});
            if (D[e] == node && !(dir == EdgeDirection::Both && S[e] == node)) in.push_back({S[e], D[e], (uint64_t)e});
        }
        std::sort(out.begin(), out.end(), [](const Edge &a, const Edge &b) { return a.dst != b.dst ? a.dst < b.dst : a.id < b.id; });
        std::sort(in.begin(), in.end(), [](const Edge &a, const Edge &b) { return a.src != b.src ? a.src < b.src : a.id < b.id; });
        std::vector<Edge> r;
        if (dir != EdgeDirection::Incoming) r = out;
        if (dir != EdgeDirection::Outgoing) r.insert(r.end(), in.begin(), in.end());
        return r;
    }
};
// every result of MATCH (a)-[*lo..hi]-(b) over the given start nodes: (from, to, path length)
static std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> vl_all(const ListAdjacency &g, const std::vector<uint64_t> &starts, uint64_t lo,
                                                                      uint64_t hi, bool rev, bool bi, int64_t dest = -1) {
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> out;
    for (uint64_t s : starts) {
        VarLenIterT<ListAdjacency> it(g, lo, hi, rev, bi, dest, true);
        it.begin_start_node(s);
        VarLenResult r;
        while (it.next(r)) out.push_back(std::make_tuple(r.from, r.to, (uint64_t)r.edges.size()));
    }
    std::sort(out.begin(), out.end());
    return out;
}
static void t_var_len_flow_goldens() {
    const uint64_t INF = UINT64_MAX;
    typedef std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> Rows;
    // test_variable_length_traversals.py:16-37: A -> B -> C -> D ("A can reach 3 nodes, B can reach 2 nodes, C can reach 1 node")
    ListAdjacency chain{{0, 1, 2}, {1, 2, 3}};
    std::vector<uint64_t> all4{0, 1, 2, 3};
    REQUIRE(vl_all(chain, all4, 1, INF, false, false).size() == 6, "test02: (a)-[*]->(b) has max_results = 6 rows");
    REQUIRE(vl_all(chain, all4, 1, INF, true, false).size() == 6, "test02: (a)<-[*]-(b) has 6 rows");
    REQUIRE(vl_all(chain, all4, 1, INF, false, true).size() == 12, "test06: the undirected traversal represents every combination twice");
    REQUIRE(vl_all(ListAdjacency{{}, {}}, all4, 0, 1, false, false).size() == 4, "test07: a zero-length traversal always returns the source");
    Rows fromA = vl_all(chain, {0}, 1, INF, false, false);
    REQUIRE((fromA == Rows{{0, 1, 1}, {0, 2, 2}, {0, 3, 3}}), "A reaches B, C, D by 1, 2, 3 hops");
    // test11_range_length_edges (:236-266): a->b, b->c, c->a, d->d; undirected patterns between a and c
    ListAdjacency tri{{0, 1, 2, 3}, {1, 2, 0, 3}};
    REQUIRE((vl_all(tri, {0}, 2, 2, false, true, 2) == Rows{{0, 2, 2}}), "(a)-[*2]-(c): length 2");
    REQUIRE((vl_all(tri, {0}, 2, INF, false, true, 2) == Rows{{0, 2, 2}}), "(a)-[*2..]-(c): length 2");
    REQUIRE((vl_all(tri, {0}, 1, INF, false, true, 2) == Rows{{0, 2, 1}, {0, 2, 2}}), "(a)-[*]-(c): lengths 1 and 2");
    REQUIRE((vl_all(tri, {3}, 0, 0, false, true) == Rows{{3, 3, 0}}), "(d)-[*0]-(): length 0");
    // test12_close_cycle (:268-293): a->b->c->a, a->d; (a)-[*2..]->(z) does not get stuck and yields z = a, c, d
    ListAdjacency cyc{{0, 1, 2, 0}, {1, 2, 0, 3}};
    Rows z = vl_all(cyc, {0}, 2, INF, false, false);
    REQUIRE((z == Rows{{0, 0, 3}, {0, 2, 2}, {0, 3, 4}}), "three results: a (3 hops), c (2), d (4)");
    // test13_fanout (:295-330): a tree with fanout 3 and depth 2; (root)-[*0..]->(n) returns all 13 nodes
    ListAdjacency tree;
    for (uint64_t a = 1; a <= 3; a++) { tree.S.push_back(0); tree.D.push_back(a); }
    for (uint64_t a = 1; a <= 3; a++) for (uint64_t k = 0; k < 3; k++) { tree.S.push_back(a); tree.D.push_back(4 + (a - 1) * 3 + k); }
    Rows t13 = vl_all(tree, {0}, 0, INF, false, false);
    REQUIRE(t13.size() == 13 && std::get<1>(t13[0]) == 0 && std::get<2>(t13[0]) == 0, "13 rows, the root first");
    std::set<uint64_t> reached;
    for (auto &r : t13) reached.insert(std::get<1>(r));
    REQUIRE(reached.size() == 13, "every node exactly once");
}

// tests/flow/test_multiple_edges.py:11-96 at the tensor level: two nodes, edges created and deleted one at a time on the same pair;
// edge counts, edge ids and the variable-length count the queries return
static void t_multiple_edges_flow() {
    Tensor t(16, 16);
    const uint64_t a = 0, b = 1;
    auto trails = [&]() {                                  // MATCH (a)-[:R*]->(b) RETURN count(b)
        t.wait();
        t.rebuild_backward();
        VarLenIter it(t, 1, UINT64_MAX, false, false, (int64_t)b, false);
        it.begin_start_node(a);
        VarLenResult r;
        uint64_t k = 0;
        while (it.next(r)) k++;
        return k;
    };
    REQUIRE(t.get(a, b).empty() && t.edge_count() == 0, "no connections yet (:16-21)");
    t.set_all_from_slices({a}, {b}, {0});
    REQUIRE((t.get(a, b) == Ids{0}) && t.edge_count() == 1, "a single edge, ID(e) = 0 (:24-36)");
    t.set_all_from_slices({a}, {b}, {1});
    REQUIRE((t.get(a, b) == Ids{0, 1}) && t.edge_count() == 2, "two connections (:39-47)");
    REQUIRE(trails() == 2, "the variable-length pattern sees both edges (:50-53)");
    auto gone = t.remove_all({std::make_tuple(0ULL, a, b)});
    REQUIRE(gone.empty() && (t.get(a, b) == Ids{1}) && t.edge_count() == 1, "first connection removed: ID(e) = 1 remains (:56-67)");
    gone = t.remove_all({std::make_tuple(1ULL, a, b)});
    REQUIRE(gone.size() == 1 && t.get(a, b).empty() && t.edge_count() == 0, "second connection removed: the pair is empty (:70-79)");
    REQUIRE(trails() == 0, "nothing left to traverse");
    t.set_all_from_slices({a}, {b}, {2});
    REQUIRE((t.get(a, b) == Ids{2}) && t.edge_count() == 1, "the connection can be re-formed (:87-95)");
    REQUIRE(trails() == 1, "one trail again");
}

static void t_traverse_over_tensor_operand() {
    uint64_t n = 64;
    Tensor t(n, n);
    t.set_all_from_slices({0, 0, 1, 2, 2, 3}, {1, 2, 3, 3, 3, 4}, {0, 1, 2, 3, 4, 5});   // (2,3) is a multi-edge pair, edge id 0 on (0,1)
    ExpandResult r1 = expand_batch({0, 2}, {TraversalMatrix(&t)}, {}, {});
    std::set<std::pair<uint64_t, uint64_t>> got, want = {{0, 1}, {0, 2}, {1, 3}};
    for (size_t k = 0; k < r1.dest.size(); k++) got.insert({r1.row_idx[k], r1.dest[k]});
    REQUIRE(got == want, "1 hop over pending tensor deltas");
    Tensor t2 = t.dup();
    t2.flush();                                                   // fold: ids now live in the committed u64 base
    t2.remove_all({std::make_tuple(0ULL, 0ULL, 1ULL)});           // tombstone the edge whose id is 0
    ExpandResult r2 = expand_batch({0}, {TraversalMatrix(&t2), TraversalMatrix(&t2), TraversalMatrix(&t2)}, {}, {});
    got.clear();
    for (size_t k = 0; k < r2.dest.size(); k++) got.insert({r2.row_idx[k], r2.dest[k]});
    want = {{0, 4}};                                              // 0 -> 2 -> 3 -> 4 ; (0,1) is gone
    REQUIRE(got == want, "3 fused hops over a dirty tensor snapshot");
}

// the coalesced form (one B200_traverse_batch_delta call) gives the per-hop delta_lmxm pairs over clean and dirty tensor operands
static void t_coalesced_traverse_over_tensor_operand() {
    auto pairs = [](const ExpandResult &r) {
        std::vector<std::pair<uint64_t, uint64_t>> v;
        for (size_t k = 0; k < r.dest.size(); k++) v.push_back({r.row_idx[k], r.dest[k]});
        return v;
    };
    uint64_t n = 256;
    std::vector<uint64_t> s, d, ids;
    for (uint64_t i = 0; i < 250; i++) { s.push_back((i * 37) % n); d.push_back((i * 101 + 7) % n); ids.push_back(i); }
    Tensor t(n, n);
    t.set_all_from_slices(s, d, ids);                             // pending: everything still in the deltas
    Tensor folded = t.dup();
    folded.flush();                                               // clean: everything in the base
    Tensor dirty = folded.dup();
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> gone;
    for (uint64_t i = 0; i < 250; i += 5) gone.push_back(std::make_tuple(ids[i], s[i], d[i]));   // (edge id, src, dst)
    dirty.remove_all(gone);                                       // tombstones over the base
    dirty.set_all_from_slices({1, 2, 3}, {200, 201, 202}, {900, 901, 902});
    VersionedMatrix lab(n, n);
    for (uint64_t v = 0; v < n; v += 3) lab.set(v, v);
    std::vector<uint64_t> src = {0, 1, 5, 9, 17, 64, 100, 255};
    for (const Tensor *x : {&t, &folded, &dirty}) {
        std::vector<TraversalMatrix> hops = {TraversalMatrix(x), TraversalMatrix(x), TraversalMatrix(&lab), TraversalMatrix(x)};
        for (bool fuse : {false, true}) {
            ExpandResult a = expand_batch(src, hops, {&lab}, {&lab}, fuse), b = expand_batch(src, hops, {&lab}, {&lab}, fuse, true);
            REQUIRE(pairs(a) == pairs(b), "coalesced tensor traversal differs from the per-hop delta_lmxm");
        }
    }
}

// multi-type hops (-[:R1|R2]->): expand_batch over a union TraversalMatrix, per hop (B200_Matrix_union_lmxm) and coalesced
// (B200_traverse_batch_union), gives the pairs of the reference's route, union_by_extract plus a hop by the fresh matrix
static void t_union_traverse_over_tensor_types() {   // device
    auto pairs = [](const ExpandResult &r) {
        std::vector<std::pair<uint64_t, uint64_t>> v;
        for (size_t k = 0; k < r.dest.size(); k++) v.push_back({r.row_idx[k], r.dest[k]});
        return v;
    };
    const uint64_t n = 64;
    auto make = [&](uint64_t mul, uint64_t add, uint64_t id, uint64_t del) {
        Tensor t(n, n);
        std::vector<uint64_t> S, D, I;
        for (uint64_t i = 0; i < 280; i++) { S.push_back((i * mul) % n); D.push_back((i * add + 7 + i / n) % n); I.push_back(id++); }
        t.set_all_from_slices(S, D, I);
        t.wait();
        t.fold_oversized();                                       // the first batch becomes the committed base
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> gone;
        for (uint64_t i = del; i < 280; i += 4) gone.push_back(std::make_tuple(I[i], S[i], D[i]));
        t.remove_all(gone);                                       // tombstones over the base
        t.set_all_from_slices({1, 2, 3, S[0]}, {50, 51, 52, D[0]}, {id, id + 1, id + 2, id + 3});   // adds, one re-add
        return t;
    };
    // c holds a's pairs but deletes others: a pair deleted in one type stays through the other, in both directions
    Tensor a = make(37, 101, 0, 0), b = make(53, 89, 10000, 1), c = make(37, 101, 20000, 2);
    VersionedMatrix lab(n, n);
    for (uint64_t v = 0; v < n; v += 3) lab.set(v, v);
    std::vector<uint64_t> src = {0, 1, 5, 9, 17, 40, 63};
    for (const std::vector<const Tensor *> &types : {std::vector<const Tensor *>{&a}, std::vector<const Tensor *>{&a, &b},
                                                     std::vector<const Tensor *>{&a, &b, &c}}) {
        VersionedMatrix u = union_by_extract(types);
        std::vector<TraversalMatrix> hops = {TraversalMatrix(&a), TraversalMatrix(types), TraversalMatrix(&lab), TraversalMatrix(types)};
        std::vector<TraversalMatrix> ref = {TraversalMatrix(&a), TraversalMatrix(&u), TraversalMatrix(&lab), TraversalMatrix(&u)};
        for (bool fuse : {false, true}) {
            ExpandResult want = expand_batch(src, ref, {}, {&lab}, fuse);
            REQUIRE(!want.dest.empty(), "test setup: the traversal finds nothing");
            REQUIRE(pairs(expand_batch(src, hops, {}, {&lab}, fuse)) == pairs(want), "per-hop union traversal differs from union_by_extract");
            REQUIRE(pairs(expand_batch(src, hops, {}, {&lab}, fuse, true)) == pairs(want), "coalesced union traversal differs from union_by_extract");
        }
    }
}

// var_len_reach (one B200_reach_batch_delta call) against the DISTINCT nodes the trail DFS reaches, over tensors whose inserts,
// deletes, re-adds, multi-edges and self-loops still sit in the deltas.  The graphs are sparse so that the DFS stays small.
struct TensorsAdjacency {       // get_node_relationships_by_type over several types
    std::vector<const Tensor *> ts;
    std::vector<Edge> operator()(uint64_t node, EdgeDirection dir) const {
        std::vector<Edge> out;
        for (const Tensor *t : ts) { std::vector<Edge> e = node_relationships(*t, node, dir); out.insert(out.end(), e.begin(), e.end()); }
        return out;
    }
};
static void t_var_len_reach_matches_trails() {   // device
    const uint64_t n = 750, used = 740;              // vertices 740.. have no edges
    uint64_t x = 4242;
    auto rnd = [&]() { x = x * 6364136223846793005ULL + 1442695040888963407ULL; return x >> 33; };
    std::vector<uint64_t> starts;
    auto make = [&](uint64_t id) {
        Tensor t(n, n);
        std::vector<uint64_t> S, D, I;
        for (uint64_t k = 0; k < 320; k++) { S.push_back(rnd() % used); D.push_back(rnd() % used); I.push_back(id++); }
        for (uint64_t v = 0; v < used; v += 61) { S.push_back(v); D.push_back(v); I.push_back(id++); }   // self-loops
        t.set_all_from_slices(S, D, I);
        t.wait();
        t.fold_oversized();                              // the first batch becomes the committed base
        REQUIRE(t.fwd_m().nvals() >= 300 && t.fwd_dp().nvals() == 0, "test setup: the first batch was folded into the base");
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rm;
        for (size_t k = 0; k < S.size(); k += 6) rm.push_back(std::make_tuple(I[k], S[k], D[k]));     // deletes from the base
        t.remove_all(rm);
        std::vector<uint64_t> S2, D2, I2;
        for (size_t k = 0; k < rm.size(); k += 3) { S2.push_back(std::get<1>(rm[k])); D2.push_back(std::get<2>(rm[k])); I2.push_back(id++); }  // re-adds
        for (uint64_t k = 0; k < 30; k++) { S2.push_back(rnd() % used); D2.push_back(rnd() % used); I2.push_back(id++); }                 // new edges
        for (size_t k = 1; k < 40; k += 13) { S2.push_back(S[k]); D2.push_back(D[k]); I2.push_back(id++); }      // a second edge on base pairs
        S2.push_back(S2[0]); D2.push_back(D2[0]); I2.push_back(id++);                                            // a pair born multi
        S2.push_back(3); D2.push_back(3); I2.push_back(id++);                                                    // a new self-loop
        t.set_all_from_slices(S2, D2, I2);
        t.wait();
        REQUIRE(t.fwd_dp().nvals() > 0 && t.fwd_dm().nvals() > 0, "test setup: the forward deltas are not empty");
        for (size_t k = 0; k < 40; k += 4) starts.push_back(S[k]);
        return t;
    };
    Tensor a = make(0), b = make(100000);
    starts.push_back(741); starts.push_back(3); starts.push_back(748);
    typedef std::set<std::pair<uint64_t, uint64_t>> Pairs;
    for (const std::vector<const Tensor *> &types : {std::vector<const Tensor *>{&a}, std::vector<const Tensor *>{&a, &b}})
        for (EdgeDirection dir : {EdgeDirection::Outgoing, EdgeDirection::Incoming})
            for (uint64_t lo : {0ULL, 1ULL})
                for (uint64_t hi : {1ULL, 2ULL, 3ULL, (unsigned long long)UINT64_MAX}) {
                    Matrix<bool> R = var_len_reach(types, dir, starts, lo, hi);
                    Pairs got, want;
                    auto it = R.iter();
                    std::tuple<uint64_t, uint64_t> e;
                    while (it.next(e)) got.insert({std::get<0>(e), std::get<1>(e)});
                    for (size_t i = 0; i < starts.size(); i++) {
                        VarLenIterT<TensorsAdjacency> dfs(TensorsAdjacency{types}, lo, hi, dir == EdgeDirection::Incoming, false, -1, false);
                        dfs.begin_start_node(starts[i]);
                        VarLenResult r;
                        while (dfs.next(r)) want.insert({(uint64_t)i, dir == EdgeDirection::Incoming ? r.from : r.to});
                    }
                    REQUIRE(got == want && R.nrows() == starts.size(), "reach differs from the trail DFS: types " << types.size() << " dir "
                            << (int)dir << " min " << lo << " max " << hi << " (" << got.size() << " vs " << want.size() << " pairs)");
                    REQUIRE(hi != 3 || lo != 1 || dir != EdgeDirection::Outgoing || want.size() >= 8, "test setup: the starts reach something");
                }
    for (auto bad : {std::make_pair(EdgeDirection::Both, 1ULL), std::make_pair(EdgeDirection::Outgoing, 2ULL)}) {
        bool threw = false;
        try { var_len_reach({&a}, bad.first, starts, bad.second, 3); } catch (const std::invalid_argument &) { threw = true; }
        REQUIRE(threw, "a bidirectional pattern or min_hops > 1 keeps the DFS");
    }
}

// var_len_reach_both (one B200_var_len_reach_both call) against the DISTINCT nodes the trail DFS reaches under Both, over the same
// kind of tensors: self-loops in the base and in dp, deleted ones, multi-edge pairs, reciprocal pairs, a pair shared by two types.
static void t_var_len_reach_both_matches_trails() {   // device
    const uint64_t n = 750, used = 740;              // vertices 740.. have no edges
    uint64_t x = 777;
    auto rnd = [&]() { x = x * 6364136223846793005ULL + 1442695040888963407ULL; return x >> 33; };
    std::vector<uint64_t> starts;
    auto make = [&](uint64_t id) {
        Tensor t(n, n);
        std::vector<uint64_t> S, D, I;
        for (uint64_t k = 0; k < 320; k++) { S.push_back(rnd() % used); D.push_back(rnd() % used); I.push_back(id++); }
        for (uint64_t v = 0; v < used; v += 37) { S.push_back(v); D.push_back(v); I.push_back(id++); }   // self-loops
        S.push_back(10); D.push_back(11); I.push_back(id++);                                               // a reciprocal pair
        S.push_back(11); D.push_back(10); I.push_back(id++);
        t.set_all_from_slices(S, D, I);
        t.wait();
        t.fold_oversized();
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rm;
        for (size_t k = 0; k < S.size(); k += 6) rm.push_back(std::make_tuple(I[k], S[k], D[k]));     // deletes from the base
        t.remove_all(rm);
        std::vector<uint64_t> S2, D2, I2;
        for (size_t k = 0; k < rm.size(); k += 3) { S2.push_back(std::get<1>(rm[k])); D2.push_back(std::get<2>(rm[k])); I2.push_back(id++); }
        for (uint64_t k = 0; k < 30; k++) { S2.push_back(rnd() % used); D2.push_back(rnd() % used); I2.push_back(id++); }
        for (size_t k = 1; k < 40; k += 13) { S2.push_back(S[k]); D2.push_back(D[k]); I2.push_back(id++); }   // multi-edge pairs
        S2.push_back(5); D2.push_back(5); I2.push_back(id++);                                                 // a new self-loop
        t.set_all_from_slices(S2, D2, I2);
        t.wait();
        REQUIRE(t.fwd_dp().nvals() > 0 && t.fwd_dm().nvals() > 0, "test setup: the forward deltas are not empty");
        for (size_t k = 0; k < 40; k += 4) starts.push_back(S[k]);
        return t;
    };
    Tensor a = make(0), b = make(100000);
    for (uint64_t s : {741ULL, 5ULL, 10ULL, 37ULL, 749ULL, 5ULL}) starts.push_back(s);
    typedef std::set<std::pair<uint64_t, uint64_t>> Pairs;
    for (const std::vector<const Tensor *> &types : {std::vector<const Tensor *>{&a}, std::vector<const Tensor *>{&a, &b}})
        for (uint64_t lo : {0ULL, 1ULL})
            for (uint64_t hi : {0ULL, 1ULL, 2ULL, 3ULL, 4ULL}) {
                Matrix<bool> R = var_len_reach_both(types, starts, lo, hi);
                Pairs got, want;
                auto it = R.iter();
                std::tuple<uint64_t, uint64_t> e;
                while (it.next(e)) got.insert({std::get<0>(e), std::get<1>(e)});
                for (size_t i = 0; i < starts.size(); i++) {
                    VarLenIterT<TensorsAdjacency> dfs(TensorsAdjacency{types}, lo, hi, false, true, -1, false);
                    dfs.begin_start_node(starts[i]);
                    VarLenResult r;
                    while (dfs.next(r)) want.insert({(uint64_t)i, r.to});
                }
                REQUIRE(got == want && R.nrows() == starts.size(), "bidirectional reach differs from the trail DFS: types " << types.size()
                        << " min " << lo << " max " << hi << " (" << got.size() << " vs " << want.size() << " pairs)");
                REQUIRE(hi != 3 || lo != 1 || want.size() >= 40, "test setup: the starts reach something");
            }
    bool threw = false;
    try { var_len_reach_both({&a}, starts, 2, 3); } catch (const std::invalid_argument &) { threw = true; }
    REQUIRE(threw, "min_hops > 1 keeps the DFS");
}

// ---- the C-compatible RDB form of a Tensor (tensor.rs:1049-1204) and of a VersionedMatrix (versioned_matrix.rs:1082-1113) ----
typedef std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> EdgeList;
static EdgeList sorted_edges(const Tensor &t) {
    EdgeList e = t.iter_edges();
    std::sort(e.begin(), e.end());
    return e;
}
static Matrix<uint64_t> valued(uint64_t n, const EdgeList &entries) {
    Matrix<uint64_t> m(n, n);
    for (auto &e : entries) m.set(std::get<0>(e), std::get<1>(e), std::get<2>(e));
    m.wait();
    return m;
}
// a stream laid out the way C FalkorDB writes a tensor: (count | MSB) in the forward matrix for a multi-edge pair, its ids as the
// INDICES of a BOOL vector blob in the base group
static Stream c_written_stream(uint64_t n, const EdgeList &fm, const EdgeList &dp, const std::vector<std::pair<uint64_t, uint64_t>> &dm,
                               uint64_t total, const std::vector<std::tuple<uint64_t, uint64_t, std::vector<uint64_t>>> &base_group,
                               const std::vector<std::tuple<uint64_t, uint64_t, std::vector<uint64_t>>> &dp_group) {
    Stream w;
    encode_matrix(valued(n, fm), w);
    encode_matrix(valued(n, dp), w);
    Matrix<bool> d(n, n);
    for (auto &e : dm) d.set(e.first, e.second, true);
    d.wait();
    encode_matrix(d, w);
    w.write_unsigned(total);
    if (!total) return w;
    for (auto *g : {&base_group, &dp_group}) {
        w.write_unsigned(g->size());
        for (auto &mp : *g) {
            w.write_unsigned(std::get<0>(mp));
            w.write_unsigned(std::get<1>(mp));
            encode_id_blob(std::get<2>(mp), GrB_INDEX_MAX_, w);
        }
    }
    return w;
}
static void t_tensor_decodes_the_c_written_form() {            // host-resident matrices only: runs without a device
    const uint64_t MSB = Tensor::MSB_MASK, BIG = ((uint64_t)1 << 40) + 1;
    Stream s = c_written_stream(8, {{0, 1, 5}, {0, 2, 0}, {1, 2, 3 | MSB}, {3, 3, 2 | MSB}, {7, 0, 42}}, {}, {}, 8,
                                {{1, 2, {7, 900, BIG}}, {3, 3, {11, 12}}}, {});
    Tensor t = Tensor::decode(s);
    REQUIRE(s.empty(), "decode consumes the whole stream");
    REQUIRE(t.get(0, 1) == Ids{5} && t.get(0, 2) == Ids{0} && t.get(7, 0) == Ids{42}, "single-edge pairs carry their id inline (0 included)");
    REQUIRE((t.get(1, 2) == Ids{7, 900, BIG}) && (t.get(3, 3) == Ids{11, 12}), "multi-edge ids are the blob's indices, ascending");
    REQUIRE(t.get(2, 2).empty() && t.get(1, 3).empty(), "absent pairs");
    uint64_t v = 0;
    REQUIRE(t.eff_get(1, 2, &v) && v == MULTI_EDGE, "a multi-edge pair holds the sentinel inline, not the count");
    REQUIRE(t.has_multi_edge() && t.multi_pairs() == 2 && t.edge_count() == 8, "2 multi-edge pairs, 8 edges");
    REQUIRE(t.matrix_t().nrows() == 0, "the backward matrix is left for rebuild_backward");
    // and back out: same layout, deltas folded (two empty layers), ids as indices
    Stream w;
    t.encode(w);
    Stream probe = w;
    Matrix<uint64_t> fm = decode_matrix<uint64_t>(probe), fdp = decode_matrix<uint64_t>(probe);
    Matrix<bool> fdm = decode_matrix<bool>(probe);
    REQUIRE(fm.nrows() == 8 && fm.ncols() == 8 && fm.nvals() == 5 && fdp.nvals() == 0 && fdm.nvals() == 0, "base holds everything");
    REQUIRE(fm.get(1, 2, &v) && v == (3 | MSB), "(count | MSB) for a multi-edge pair");
    REQUIRE(fm.get(3, 3, &v) && v == (2 | MSB) && fm.get(0, 2, &v) && v == 0 && fm.get(7, 0, &v) && v == 42, "forward values");
    REQUIRE(probe.read_unsigned() == 8 && probe.read_unsigned() == 2, "total edges, base group size");
    REQUIRE(probe.read_unsigned() == 1 && probe.read_unsigned() == 2 && (decode_id_blob(probe) == Ids{7, 900, BIG}), "first pair");
    REQUIRE(probe.read_unsigned() == 3 && probe.read_unsigned() == 3 && (decode_id_blob(probe) == Ids{11, 12}), "second pair");
    REQUIRE(probe.read_unsigned() == 0 && probe.empty(), "empty delta-plus group ends the stream");
    Tensor t2 = Tensor::decode(w);
    REQUIRE(sorted_edges(t2) == sorted_edges(t) && t2.edge_count() == 8, "encode -> decode keeps every (src, dst, id)");
    // defensive merge of on-disk deltas: (m \ dm) U dp, ids from both groups
    Stream s2 = c_written_stream(8, {{0, 1, 5}, {7, 0, 42}, {4, 4, 9}}, {{7, 0, 43}, {6, 6, 2 | MSB}}, {{7, 0}, {0, 1}}, 4, {},
                                 {{6, 6, {100, 101}}});
    Tensor t3 = Tensor::decode(s2);
    REQUIRE(t3.get(7, 0) == Ids{43} && t3.get(0, 1).empty() && t3.get(4, 4) == Ids{9} && (t3.get(6, 6) == Ids{100, 101}), "merged deltas");
    // an empty tensor: three empty layers and a zero count
    Tensor e(5, 5);
    Stream we;
    e.encode(we);
    REQUIRE(we.items.size() == 3 * 26 + 1 && we.items.back().u == 0, "3 x (container + 5 payload vectors x 5 items) + total 0");
    Tensor e2 = Tensor::decode(we);
    REQUIRE(e2.edge_count() == 0 && e2.fwd_m().nrows() == 5, "empty round trip");
    // malformed input surfaces as an error, never as a half-built tensor
    Stream bad = c_written_stream(8, {{0, 1, 5}}, {}, {}, 1, {}, {});
    bad.items.pop_back();
    bool threw = false;
    try { Tensor::decode(bad); } catch (const std::runtime_error &) { threw = true; }
    REQUIRE(threw, "a truncated tensor section is an error");
    Stream tiny;
    tiny.write_buffer("abc", 3);
    threw = false;
    try { Tensor::decode(tiny); } catch (const std::runtime_error &ex) { threw = std::string(ex.what()).find("container buffer too small") != std::string::npos; }
    REQUIRE(threw, "container buffer too small");
}
static void t_tensor_encode_decode_after_mutations() {          // device: batched inserts, a fold, bulk deletes, backward rebuild
    Tensor t(64, 64);
    std::map<std::pair<uint64_t, uint64_t>, std::set<uint64_t>> model;       // what the tensor must hold, kept independently
    uint64_t next = 0;
    std::vector<uint64_t> S, D, I;
    auto edge = [&](uint64_t s, uint64_t d) { S.push_back(s); D.push_back(d); I.push_back(next); model[{s, d}].insert(next); next++; };
    auto at = [&](uint64_t a, uint64_t b) -> std::set<uint64_t> & { return model[std::make_pair(a, b)]; };
    auto commit = [&]() { t.set_all_from_slices(S, D, I); S.clear(); D.clear(); I.clear(); };
    auto expected = [&]() {
        EdgeList e;
        for (auto &kv : model) for (uint64_t id : kv.second) e.push_back(std::make_tuple(kv.first.first, kv.first.second, id));
        std::sort(e.begin(), e.end());
        return e;
    };
    for (uint64_t s = 0; s < 64; s++) for (uint64_t k = 1; k <= 5; k++) edge(s, (s * 7 + k * 5) % 64);   // 320 distinct pairs, id 0 included
    commit();
    t.wait();
    t.fold_oversized();                                          // 320 >= MIN_FOLD_DELTA and dominates the empty base: dp folds into m
    REQUIRE(t.fwd_m().nvals() == 320 && t.fwd_dp().nvals() == 0, "the first batch was folded into the base");
    edge(2, 19); edge(2, 19);                                    // (2,19) holds id 10 in the base: promoted to three edges
    edge(50, 51); edge(50, 51);                                  // a pair born multi inside one batch
    edge(60, 1); edge(60, 1); edge(61, 2);
    commit();
    REQUIRE(at(2, 19).size() == 3 && *at(2, 19).begin() == 10, "test setup: (2,19) was a base single (id 10)");
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rm;
    auto drop = [&](uint64_t s, uint64_t d, uint64_t id) {
        rm.push_back(std::make_tuple(id, s, d));
        auto it = model.find({s, d});
        it->second.erase(id);
        if (it->second.empty()) model.erase(it);
    };
    for (uint64_t s = 10; s < 20; s++) drop(s, (s * 7 + 10) % 64, s * 5 + 1);        // ten singles out of the base (k = 2)
    drop(2, 19, *at(2, 19).rbegin());                       // one of (2,19)'s three
    drop(60, 1, *at(60, 1).begin());                        // (60,1) down to one edge: demoted to inline
    t.remove_all(rm);
    t.wait();
    EdgeList before = sorted_edges(t);
    uint64_t count = t.edge_count();
    REQUIRE(before == expected(), "the tensor holds what the model holds before encoding");
    REQUIRE(count == before.size(), "edge_count agrees with the enumeration");
    REQUIRE(t.fwd_dm().nvals() >= 10 && t.fwd_dp().nvals() > 0, "test setup: all three forward layers are populated");
    Stream w;
    t.encode(w);
    REQUIRE(sorted_edges(t) == before, "encode leaves the tensor usable");
    Stream probe = w;
    Matrix<uint64_t> fm = decode_matrix<uint64_t>(probe), fdp = decode_matrix<uint64_t>(probe);
    Matrix<bool> fdm = decode_matrix<bool>(probe);
    REQUIRE(fm.nvals() == model.size() && fdp.nvals() == 0 && fdm.nvals() == 0, "deltas are folded on the way out");
    REQUIRE(probe.read_unsigned() == count, "total edge count");
    uint64_t v = 0;
    REQUIRE(fm.get(2, 19, &v) && v == (2 | Tensor::MSB_MASK) && fm.get(50, 51, &v) && v == (2 | Tensor::MSB_MASK), "(count | MSB)");
    REQUIRE(fm.get(60, 1, &v) && v == *at(60, 1).begin() && fm.get(0, 5, &v) && v == 0, "inline ids, edge id 0 included");
    Tensor u = Tensor::decode(w);
    u.rebuild_backward();
    REQUIRE(sorted_edges(u) == before && u.edge_count() == count, "every (src, dst, id) survives");
    for (auto &kv : model) {
        Ids want(kv.second.begin(), kv.second.end());
        REQUIRE(u.get(kv.first.first, kv.first.second) == want, "ids of (" << kv.first.first << "," << kv.first.second << ")");
    }
    REQUIRE(u.multi_pairs() == 2 && u.matrix_t().nvals() == model.size() && u.matrix_t().get(19, 2) && u.matrix_t().get(51, 50) &&
            !u.matrix_t().get((10 * 7 + 10) % 64, 10), "backward = transpose of the live pattern");
    // the decoded tensor keeps working as an edge store
    std::vector<uint64_t> S3 = {2}, D3 = {19}, I3 = {next};
    u.set_all_from_slices(S3, D3, I3);
    REQUIRE(u.get(2, 19).size() == 3 && u.get(2, 19).back() == next && u.edge_count() == count + 1, "insert after decode");
}
static void t_tensor_bulk_load_matches_set_all_from_slices() {  // device
    const uint64_t n = 128;
    std::vector<uint64_t> S, D, I;
    uint64_t x = 12345;
    auto rnd = [&]() { x = x * 6364136223846793005ULL + 1442695040888963407ULL; return x >> 33; };
    const uint64_t count = 3000;
    for (uint64_t k = 0; k < count; k++) {
        bool hot = rnd() % 4 == 0;                               // a quarter of the edges land on 40 hot pairs: long id lists
        S.push_back(hot ? rnd() % 5 : rnd() % n);
        D.push_back(hot ? rnd() % 8 : rnd() % n);
        I.push_back((k * 7919) % count);                         // a permutation of 0..count-1 (7919 is prime to 3000): ids arrive unordered, 0 included
    }
    std::map<std::pair<uint64_t, uint64_t>, std::set<uint64_t>> model;
    for (uint64_t k = 0; k < count; k++) model[std::make_pair(S[k], D[k])].insert(I[k]);
    Tensor a(n, n);
    a.set_all_from_slices(S, D, I);
    a.wait();
    Tensor b = Tensor::bulk_load(n, n, S, D, I);
    REQUIRE(sorted_edges(b) == sorted_edges(a) && sorted_edges(b).size() == count, "same (src, dst, id) set as the reference's insert loop");
    uint64_t multi = 0, v = 0;
    for (auto &kv : model) {
        Ids want(kv.second.begin(), kv.second.end());
        REQUIRE(b.get(kv.first.first, kv.first.second) == want, "ids of (" << kv.first.first << "," << kv.first.second << ")");
        REQUIRE(b.fwd_m().get(kv.first.first, kv.first.second, &v) && v == (want.size() > 1 ? MULTI_EDGE : want[0]), "inline value");
        multi += want.size() > 1;
    }
    REQUIRE(multi > 40 && b.multi_pairs() == multi && a.multi_pairs() == multi, "multi-edge pairs");
    REQUIRE(b.edge_count() == count && a.edge_count() == count, "edge_count");
    REQUIRE(b.fwd_m().nvals() == model.size() && b.fwd_dp().nvals() == 0 && b.fwd_dm().nvals() == 0, "everything in the base, no deltas");
    REQUIRE(b.matrix_t().nvals() == model.size() && b.extract().nvals() == model.size(), "backward matrix and pattern");
    {
        auto it = b.matrix_t().iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) REQUIRE(model.count(std::make_pair(std::get<1>(t), std::get<0>(t))), "backward entry without a forward pair");
    }
    // the loaded tensor is an ordinary tensor afterwards
    std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rm;
    auto first = model.begin();
    for (uint64_t id : first->second) rm.push_back(std::make_tuple(id, first->first.first, first->first.second));
    b.remove_all(rm);
    REQUIRE(b.get(first->first.first, first->first.second).empty() && b.edge_count() == count - first->second.size(), "delete after load");
    // corner cases
    Tensor e = Tensor::bulk_load(n, n, {}, {}, {});
    REQUIRE(e.edge_count() == 0 && e.fwd_m().nrows() == n, "empty load");
    bool threw = false;
    try { Tensor::bulk_load(n, n, {1}, {n}, {0}); } catch (const std::runtime_error &) { threw = true; }
    REQUIRE(threw, "an endpoint outside the matrix is an error");
}
static void t_versioned_matrix_encode_decode() {
    VersionedMatrix v(40, 40);
    for (uint64_t k = 0; k < 30; k++) v.set(k, (k * 3) % 40);
    v.wait();
    v.remove(3, 9);
    v.set(39, 39);
    std::vector<std::tuple<uint64_t, uint64_t>> want, got;
    {
        auto it = v.iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) want.push_back(t);
    }
    Stream w;
    v.encode(w);
    REQUIRE(w.items.size() == 3 * 26, "three layers: container + 5 payload vectors each");
    VersionedMatrix u = VersionedMatrix::decode(w);
    REQUIRE(w.empty() && u.nvals() == v.nvals() && u.nrows() == 40, "layers in order");
    {
        auto it = u.iter();
        std::tuple<uint64_t, uint64_t> t;
        while (it.next(t)) got.push_back(t);
    }
    REQUIRE(got == want && got.size() == 30 && u.get(39, 39) && !u.get(3, 9), "effective content");
    u.set(3, 9);
    REQUIRE(u.nvals() == 31, "usable after decode");
}

struct TestEntry { const char *name; void (*fn)(); };
static TestEntry TESTS[] = {
    {"read_path_balance_point_is_flat_in_base_size", t_read_path_balance_point_is_flat_in_base_size},
    {"write_path_is_16x_looser_than_read_path", t_write_path_is_16x_looser_than_read_path},
    {"balance_point_grows_as_sqrt_of_transaction_size", t_balance_point_grows_as_sqrt_of_transaction_size},
    {"delta_comparable_to_base_always_folds", t_delta_comparable_to_base_always_folds},
    {"tiny_deltas_and_read_only_transactions_never_fold", t_tiny_deltas_and_read_only_transactions_never_fold},
    {"delta_invariants_hold_across_mutation_sequences", t_delta_invariants_hold_across_mutation_sequences},
    {"folded_entry_deleted_and_re_added_stays_out_of_dp", t_folded_entry_deleted_and_re_added_stays_out_of_dp},
    {"motogp_two_hop", t_motogp_two_hop},
    {"multi_pairs_after_within_batch_duplicates", t_multi_pairs_after_within_batch_duplicates},
    {"multi_pairs_matches_the_sentinel_count", t_multi_pairs_matches_the_sentinel_count},
    {"bulk_remove_and_extract_edge_id_zero", t_bulk_remove_and_extract_edge_id_zero},
    {"deleting_everything_folds_the_tombstones_away", t_deleting_everything_folds_the_tombstones_away},
    {"batch_demote_leaves_every_survivor_inline", t_batch_demote_leaves_every_survivor_inline},
    {"batch_can_demote_and_then_empty_the_same_pair", t_batch_can_demote_and_then_empty_the_same_pair},
    {"demoting_to_the_committed_value_cancels_to_clean", t_demoting_to_the_committed_value_cancels_to_clean},
    {"traverse_over_tensor_operand", t_traverse_over_tensor_operand},
    {"coalesced_traverse_over_tensor_operand", t_coalesced_traverse_over_tensor_operand},
    {"var_len_reach_matches_trails", t_var_len_reach_matches_trails},
    {"var_len_reach_both_matches_trails", t_var_len_reach_both_matches_trails},
    {"union_traverse_over_tensor_types", t_union_traverse_over_tensor_types},
    {"repack_output_batches", t_repack_output_batches},
    {"repack_logic", t_repack_logic},
    {"var_len_trails", t_var_len_trails},
    {"var_len_trails_logic", t_var_len_trails_logic},
    {"var_len_types_labels_logic", t_var_len_types_labels_logic},
    {"var_len_flow_goldens", t_var_len_flow_goldens},
    {"multiple_edges_flow", t_multiple_edges_flow},
    {"tensor_decodes_the_c_written_form", t_tensor_decodes_the_c_written_form},
    {"tensor_encode_decode_after_mutations", t_tensor_encode_decode_after_mutations},
    {"versioned_matrix_encode_decode", t_versioned_matrix_encode_decode},
    {"tensor_bulk_load_matches_set_all_from_slices", t_tensor_bulk_load_matches_set_all_from_slices},
};

extern "C" {

const char *fdbh_last_message(void) { return g_msg.c_str(); }

// run one transcribed reference unit test by name; 0 = pass
int fdbh_run_test(const char *name) {
    for (auto &t : TESTS)
        if (!strcmp(t.name, name)) {
            try { GxB_init(GrB_NONBLOCKING, nullptr, nullptr, nullptr, nullptr); t.fn(); g_msg = "ok"; return 0; }
            catch (const std::exception &e) { g_msg = e.what(); return 1; }
        }
    g_msg = "unknown test";
    return 2;
}
// the tensor.rs tests whose writes can take either route; write_dev 1: through the device plans
static const char *WRITE_TESTS[] = {"multi_pairs_after_within_batch_duplicates", "multi_pairs_matches_the_sentinel_count",
                                    "bulk_remove_and_extract_edge_id_zero", "deleting_everything_folds_the_tombstones_away",
                                    "batch_demote_leaves_every_survivor_inline", "batch_can_demote_and_then_empty_the_same_pair",
                                    "demoting_to_the_committed_value_cancels_to_clean"};
int fdbh_run_write_test(const char *name, int write_dev) {
    bool known = false;
    for (const char *w : WRITE_TESTS) known = known || !strcmp(w, name);
    if (!known) { g_msg = "not a write-route test"; return 2; }
    g_write_dev = write_dev != 0;
    int rc = fdbh_run_test(name);
    g_write_dev = false;
    return rc;
}

void *fdbh_vm_from_csr(uint64_t nrows, uint64_t ncols, const uint64_t *Ap, const uint32_t *Aj) {
    try {
        GrB_Matrix raw = nullptr;
        grb_ok(B200_Matrix_import_CSR(&raw, GrB_BOOL, nrows, ncols, Ap, Aj, nullptr, B200_LOC_HOST), "import_CSR");
        return new VersionedMatrix(VersionedMatrix::from_matrix(Matrix<bool>::adopt(raw, false)));
    } catch (const std::exception &e) { g_msg = e.what(); return nullptr; }
}
void *fdbh_vm_new(uint64_t nrows, uint64_t ncols) {
    try { return new VersionedMatrix(nrows, ncols); } catch (const std::exception &e) { g_msg = e.what(); return nullptr; }
}
void fdbh_vm_free(void *vm) { delete (VersionedMatrix *)vm; }
int fdbh_vm_set(void *vm, uint64_t i, uint64_t j) { try { ((VersionedMatrix *)vm)->set(i, j); return 0; } catch (const std::exception &e) { g_msg = e.what(); return 1; } }
int fdbh_vm_remove(void *vm, uint64_t i, uint64_t j) { try { ((VersionedMatrix *)vm)->remove(i, j); return 0; } catch (const std::exception &e) { g_msg = e.what(); return 1; } }
int64_t fdbh_vm_nvals(void *vm) { try { return (int64_t)((VersionedMatrix *)vm)->nvals(); } catch (const std::exception &e) { g_msg = e.what(); return -1; } }

// CondTraverse batched path.  Outputs are malloc'ed; free with fdbh_free.
static int expand_batch_c(const uint64_t *src_ids, uint64_t nsrc, void **hops, uint64_t nhops, void **src_labels, uint64_t nsl,
                          void **dst_labels, uint64_t ndl, uint64_t **out_rows, uint64_t **out_dest, uint64_t *nout, bool fuse,
                          bool coalesced = false) {
    try {
        std::vector<uint64_t> src(src_ids, src_ids + nsrc);
        std::vector<TraversalMatrix> h;
        std::vector<const VersionedMatrix *> sl, dl;
        for (uint64_t k = 0; k < nhops; k++) h.push_back(TraversalMatrix((const VersionedMatrix *)hops[k]));
        for (uint64_t k = 0; k < nsl; k++) sl.push_back((const VersionedMatrix *)src_labels[k]);
        for (uint64_t k = 0; k < ndl; k++) dl.push_back((const VersionedMatrix *)dst_labels[k]);
        ExpandResult r = expand_batch(src, h, sl, dl, fuse, coalesced);
        *nout = r.dest.size();
        *out_rows = (uint64_t *)malloc(sizeof(uint64_t) * (r.dest.size() + 1));
        *out_dest = (uint64_t *)malloc(sizeof(uint64_t) * (r.dest.size() + 1));
        memcpy(*out_rows, r.row_idx.data(), sizeof(uint64_t) * r.dest.size());
        memcpy(*out_dest, r.dest.data(), sizeof(uint64_t) * r.dest.size());
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
int fdbh_expand_batch(const uint64_t *src_ids, uint64_t nsrc, void **hops, uint64_t nhops, void **src_labels, uint64_t nsl,
                      void **dst_labels, uint64_t ndl, uint64_t **out_rows, uint64_t **out_dest, uint64_t *nout) {
    return expand_batch_c(src_ids, nsrc, hops, nhops, src_labels, nsl, dst_labels, ndl, out_rows, out_dest, nout, false);
}
// destination-label filters applied on the device as extra diagonal hops (SURVEY 8f-2)
int fdbh_expand_batch_fused(const uint64_t *src_ids, uint64_t nsrc, void **hops, uint64_t nhops, void **src_labels, uint64_t nsl,
                            void **dst_labels, uint64_t ndl, uint64_t **out_rows, uint64_t **out_dest, uint64_t *nout) {
    return expand_batch_c(src_ids, nsrc, hops, nhops, src_labels, nsl, dst_labels, ndl, out_rows, out_dest, nout, true);
}
// every hop (and, with fuse_dst_labels, every destination label) in one B200_traverse_batch_delta call
int fdbh_expand_batch_coalesced(const uint64_t *src_ids, uint64_t nsrc, void **hops, uint64_t nhops, void **src_labels, uint64_t nsl,
                                void **dst_labels, uint64_t ndl, uint64_t **out_rows, uint64_t **out_dest, uint64_t *nout,
                                int fuse_dst_labels) {
    return expand_batch_c(src_ids, nsrc, hops, nhops, src_labels, nsl, dst_labels, ndl, out_rows, out_dest, nout, fuse_dst_labels != 0,
                          true);
}
// CondVarLenTraverse's reach fast path (var_len_reach): tensors are Tensor pointers, dir 0 outgoing / 1 incoming, max_hops
// UINT64_MAX unbounded.  Output: the (row, node) pairs in row order, malloc'ed; free with fdbh_free.
int fdbh_var_len_reach(void **tensors, uint64_t ntypes, int dir, const uint64_t *starts, uint64_t nstarts, uint64_t min_hops,
                       uint64_t max_hops, uint64_t **out_rows, uint64_t **out_nodes, uint64_t *nout) {
    try {
        std::vector<const Tensor *> types;
        for (uint64_t k = 0; k < ntypes; k++) types.push_back((const Tensor *)tensors[k]);
        if (dir != 0 && dir != 1) throw std::invalid_argument("var_len_reach: dir must be 0 (outgoing) or 1 (incoming)");
        Matrix<bool> R = var_len_reach(types, dir == 0 ? EdgeDirection::Outgoing : EdgeDirection::Incoming,
                                       std::vector<uint64_t>(starts, starts + nstarts), min_hops, max_hops);
        std::vector<uint64_t> rows, nodes;
        auto it = R.iter();
        std::tuple<uint64_t, uint64_t> e;
        while (it.next(e)) { rows.push_back(std::get<0>(e)); nodes.push_back(std::get<1>(e)); }
        *nout = rows.size();
        *out_rows = (uint64_t *)malloc(sizeof(uint64_t) * (rows.size() + 1));
        *out_nodes = (uint64_t *)malloc(sizeof(uint64_t) * (rows.size() + 1));
        memcpy(*out_rows, rows.data(), sizeof(uint64_t) * rows.size());
        memcpy(*out_nodes, nodes.data(), sizeof(uint64_t) * rows.size());
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
// The bidirectional counterpart (var_len_reach_both): the (row, node) pairs in row order, malloc'ed; free with fdbh_free.
int fdbh_var_len_reach_both(void **tensors, uint64_t ntypes, const uint64_t *starts, uint64_t nstarts, uint64_t min_hops,
                            uint64_t max_hops, uint64_t **out_rows, uint64_t **out_nodes, uint64_t *nout) {
    try {
        std::vector<const Tensor *> types;
        for (uint64_t k = 0; k < ntypes; k++) types.push_back((const Tensor *)tensors[k]);
        Matrix<bool> R = var_len_reach_both(types, std::vector<uint64_t>(starts, starts + nstarts), min_hops, max_hops);
        std::vector<uint64_t> rows, nodes;
        auto it = R.iter();
        std::tuple<uint64_t, uint64_t> e;
        while (it.next(e)) { rows.push_back(std::get<0>(e)); nodes.push_back(std::get<1>(e)); }
        *nout = rows.size();
        *out_rows = (uint64_t *)malloc(sizeof(uint64_t) * (rows.size() + 1));
        *out_nodes = (uint64_t *)malloc(sizeof(uint64_t) * (rows.size() + 1));
        memcpy(*out_rows, rows.data(), sizeof(uint64_t) * rows.size());
        memcpy(*out_nodes, nodes.data(), sizeof(uint64_t) * rows.size());
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
void fdbh_free(void *p) { free(p); }

// ---- a relationship Tensor for the edge-id routes: GRAPH.BULK's load, batched inserts and deletes with pending writes ----
void *fdbh_tensor_bulk_load(uint64_t n, const uint64_t *srcs, const uint64_t *dsts, const uint64_t *ids, uint64_t k) {
    try {
        return new Tensor(Tensor::bulk_load(n, n, std::vector<uint64_t>(srcs, srcs + k), std::vector<uint64_t>(dsts, dsts + k),
                                            std::vector<uint64_t>(ids, ids + k)));
    } catch (const std::exception &e) { g_msg = e.what(); return nullptr; }
}
void fdbh_tensor_free(void *t) { delete (Tensor *)t; }
int fdbh_tensor_set_all(void *t, const uint64_t *srcs, const uint64_t *dsts, const uint64_t *ids, uint64_t k) {
    try {
        ((Tensor *)t)->set_all_from_slices(std::vector<uint64_t>(srcs, srcs + k), std::vector<uint64_t>(dsts, dsts + k),
                                           std::vector<uint64_t>(ids, ids + k));
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
int fdbh_tensor_remove_all(void *t, const uint64_t *ids, const uint64_t *srcs, const uint64_t *dsts, uint64_t k) {
    try {
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rels;
        for (uint64_t q = 0; q < k; q++) rels.push_back(std::make_tuple(ids[q], srcs[q], dsts[q]));
        ((Tensor *)t)->remove_all(rels);
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
// Tensor::set_all_from_slices_dev / remove_all_dev (the device plans), and remove_all with its emptied pairs.  Emptied pairs are
// malloc'ed (free with fdbh_free): the device route lists them ascending, the reference in discovery order.
int fdbh_tensor_set_all_dev(void *t, const uint64_t *srcs, const uint64_t *dsts, const uint64_t *ids, uint64_t k) {
    try {
        ((Tensor *)t)->set_all_from_slices_dev(std::vector<uint64_t>(srcs, srcs + k), std::vector<uint64_t>(dsts, dsts + k),
                                               std::vector<uint64_t>(ids, ids + k));
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
static int remove_emptied(void *t, const uint64_t *ids, const uint64_t *srcs, const uint64_t *dsts, uint64_t k, bool dev,
                          uint64_t **out_src, uint64_t **out_dst, uint64_t *nout) {
    try {
        std::vector<std::tuple<uint64_t, uint64_t, uint64_t>> rels;
        for (uint64_t q = 0; q < k; q++) rels.push_back(std::make_tuple(ids[q], srcs[q], dsts[q]));
        auto em = dev ? ((Tensor *)t)->remove_all_dev(rels) : ((Tensor *)t)->remove_all(rels);
        *nout = em.size();
        *out_src = (uint64_t *)malloc(sizeof(uint64_t) * (em.size() + 1));
        *out_dst = (uint64_t *)malloc(sizeof(uint64_t) * (em.size() + 1));
        if (!*out_src || !*out_dst) { free(*out_src); free(*out_dst); throw std::bad_alloc(); }
        for (size_t q = 0; q < em.size(); q++) { (*out_src)[q] = em[q].first; (*out_dst)[q] = em[q].second; }
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
int fdbh_tensor_remove_all_dev(void *t, const uint64_t *ids, const uint64_t *srcs, const uint64_t *dsts, uint64_t k,
                               uint64_t **out_src, uint64_t **out_dst, uint64_t *nout) {
    return remove_emptied(t, ids, srcs, dsts, k, true, out_src, out_dst, nout);
}
int fdbh_tensor_remove_all_emptied(void *t, const uint64_t *ids, const uint64_t *srcs, const uint64_t *dsts, uint64_t k,
                                   uint64_t **out_src, uint64_t **out_dst, uint64_t *nout) {
    return remove_emptied(t, ids, srcs, dsts, k, false, out_src, out_dst, nout);
}
// the six Delta counters (dp, dm; mt's dp, dm; me's dp, dm)
int fdbh_tensor_counts(void *t, uint64_t *out6) {
    try { ((const Tensor *)t)->counts(out6); return 0; } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
void *fdbh_tensor_dup(void *t) {
    try { return new Tensor(((const Tensor *)t)->dup()); } catch (const std::exception &e) { g_msg = e.what(); return nullptr; }
}
int fdbh_tensor_fold_oversized(void *t) {
    try { ((Tensor *)t)->fold_oversized(); return 0; } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
int fdbh_tensor_flush(void *t) {
    try { ((Tensor *)t)->flush(); return 0; } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
int64_t fdbh_tensor_edge_count(void *t) {
    try { return (int64_t)((const Tensor *)t)->edge_count(); } catch (const std::exception &e) { g_msg = e.what(); return -1; }
}
// VersionedMatrix::set_all<NEW> (route 0) or set_all_dev<NEW> (route 1) over the pairs (rows[k], cols[k])
int fdbh_vm_set_all(void *vm, const uint64_t *rows, const uint64_t *cols, uint64_t k, int is_new, int route) {
    try {
        std::vector<std::pair<uint64_t, uint64_t>> e;
        for (uint64_t q = 0; q < k; q++) e.push_back({rows[q], cols[q]});
        VersionedMatrix *v = (VersionedMatrix *)vm;
        if (route == 0) { if (is_new) v->set_all<true>(e); else v->set_all<false>(e); }
        else { if (is_new) v->set_all_dev<true>(e); else v->set_all_dev<false>(e); }
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
// the two Delta counters and the three layer handles (m, dp, dm) of a VersionedMatrix, borrowed
int fdbh_vm_state(void *vm, uint64_t *out2, void **out3) {
    try {
        const VersionedMatrix *v = (const VersionedMatrix *)vm;
        v->wait_all();
        v->counts(out2);
        out3[0] = v->m().inner(); out3[1] = v->dp().inner(); out3[2] = v->dm().inner();
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
// the nine layer handles (B200_TensorLayers order) after Tensor::wait(); borrowed, valid until the tensor changes
int fdbh_tensor_layers(void *tp, void **out9) {
    try {
        const Tensor *t = (const Tensor *)tp;
        t->wait();
        const VersionedMatrix &mt = t->matrix_t(), &me = t->edge_versioned();
        mt.wait_all(); me.wait_all();
        GrB_Matrix h[9] = {t->fwd_m().inner(), t->fwd_dp().inner(), t->fwd_dm().inner(), mt.m().inner(), mt.dp().inner(),
                           mt.dm().inner(), me.m().inner(), me.dp().inner(), me.dm().inner()};
        for (int k = 0; k < 9; k++) out9[k] = h[k];
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
// The relationships of a batch of rows over Tensor pointers.  route 0: B200_expand_edges (expand_edges); 1: Tensor::get per pair
// (expand_edges_by_get, or expand_into_by_get with targets); 2: B200_traverse_batch_union then a get per pair (bind_edge's route:
// dir OUT, mode FIRST, no targets).  Outputs are malloc'ed; free with fdbh_free.
int fdbh_expand_edges(void **tensors, uint64_t ntypes, const uint64_t *srcs, const uint64_t *tgts, uint64_t n, int dir, int mode,
                      int route, uint64_t **out_p, uint32_t **out_node, uint64_t **out_edge, uint16_t **out_type, uint8_t **out_rev,
                      uint64_t *nout) {
    try {
        std::vector<const Tensor *> types;
        for (uint64_t k = 0; k < ntypes; k++) types.push_back((const Tensor *)tensors[k]);
        std::vector<uint64_t> s(srcs, srcs + n), d;
        if (tgts) d.assign(tgts, tgts + n);
        EdgeExpansion r;
        if (route == 0) r = expand_edges(s, tgts ? &d : nullptr, types, dir, mode);
        else if (route == 1) r = tgts ? expand_into_by_get(s, d, types, dir, mode) : expand_edges_by_get(s, types, dir, mode);
        else if (route == 2 && !tgts && dir == B200_DIR_OUT && mode == B200_EDGES_FIRST) r = bind_edge_after_traverse(s, types);
        else throw std::invalid_argument("expand_edges: unknown route, or route 2 outside dir OUT / mode FIRST without targets");
        const uint64_t m = r.edge.size();
        *nout = m;
        auto out = [](auto **dst, const auto &v) {
            *dst = (std::remove_reference_t<decltype(**dst)> *)malloc(sizeof(**dst) * (v.size() + 1));
            if (!*dst) throw std::bad_alloc();
            memcpy(*dst, v.data(), sizeof(**dst) * v.size());
        };
        out(out_p, r.p); out(out_node, r.node); out(out_edge, r.edge); out(out_type, r.type); out(out_rev, r.rev);
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}

// CondVarLenTraverse's trails over Tensor pointers (dir 0 out / 1 in / 2 both; dests NULL or < 0: none; labels: VersionedMatrix
// pointers, NULL = a label the graph lacks).  fdbh_var_len_trails: B200_var_len_trails (var_len_trails); fdbh_var_len_trails_dfs:
// the reference's DFS (var_len_trails_dfs).  Outputs (malloc'ed; free with fdbh_free): p[nstarts + 1]; per trail its end (the walk's
// last node) and hop count; with emit_path the edges (npath) and nodes (npath + nout) in walk order, as B200_var_len_trails lays them.
static int var_len_out(const VarLenBatch &b, EdgeDirection dir, uint64_t **out_p, uint64_t **out_end, uint64_t **out_hops,
                       uint64_t **path_edge, uint64_t **path_node, uint64_t *nout, uint64_t *npath) {
    std::vector<uint64_t> end, hops, pe, pn;
    for (const VarLenResult &r : b.r) {
        end.push_back(dir == EdgeDirection::Incoming ? r.from : r.to);
        hops.push_back(r.hops);
        pe.insert(pe.end(), r.edges.begin(), r.edges.end());
        pn.insert(pn.end(), r.nodes.begin(), r.nodes.end());
    }
    *nout = end.size(); *npath = pe.size();
    auto out = [](uint64_t **dst, const std::vector<uint64_t> &v) {
        *dst = (uint64_t *)malloc(sizeof(uint64_t) * (v.size() + 1));
        if (!*dst) throw std::bad_alloc();
        memcpy(*dst, v.data(), sizeof(uint64_t) * v.size());
    };
    out(out_p, b.p); out(out_end, end); out(out_hops, hops); out(path_edge, pe); out(path_node, pn);
    return 0;
}
static int var_len_c(bool dev, void **tensors, uint64_t ntypes, int dir, const uint64_t *starts, const int64_t *dests, uint64_t nstarts,
                     uint64_t min_hops, uint64_t max_hops, void **labels, uint64_t nlabels, int emit_path, uint64_t tree_capacity,
                     uint64_t **out_p, uint64_t **out_end, uint64_t **out_hops, uint64_t **path_edge, uint64_t **path_node,
                     uint64_t *nout, uint64_t *npath) {
    try {
        std::vector<const Tensor *> types;
        for (uint64_t k = 0; k < ntypes; k++) types.push_back((const Tensor *)tensors[k]);
        std::vector<const VersionedMatrix *> labs;
        for (uint64_t k = 0; k < nlabels; k++) labs.push_back((const VersionedMatrix *)labels[k]);
        if (dir < 0 || dir > 2) throw std::invalid_argument("var_len_trails: dir must be 0, 1 or 2");
        const EdgeDirection d = dir == 0 ? EdgeDirection::Outgoing : dir == 1 ? EdgeDirection::Incoming : EdgeDirection::Both;
        std::vector<uint64_t> s(starts, starts + nstarts);
        std::vector<int64_t> ds;
        if (dests) ds.assign(dests, dests + nstarts);
        VarLenBatch b = dev ? var_len_trails(types, d, s, ds, min_hops, max_hops, labs, emit_path != 0, tree_capacity)
                            : var_len_trails_dfs(types, d, s, ds, min_hops, max_hops, labs, emit_path != 0);
        return var_len_out(b, d, out_p, out_end, out_hops, path_edge, path_node, nout, npath);
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}
int fdbh_var_len_trails(void **tensors, uint64_t ntypes, int dir, const uint64_t *starts, const int64_t *dests, uint64_t nstarts,
                        uint64_t min_hops, uint64_t max_hops, void **labels, uint64_t nlabels, int emit_path, uint64_t tree_capacity,
                        uint64_t **out_p, uint64_t **out_end, uint64_t **out_hops, uint64_t **path_edge, uint64_t **path_node,
                        uint64_t *nout, uint64_t *npath) {
    return var_len_c(true, tensors, ntypes, dir, starts, dests, nstarts, min_hops, max_hops, labels, nlabels, emit_path, tree_capacity,
                     out_p, out_end, out_hops, path_edge, path_node, nout, npath);
}
int fdbh_var_len_trails_dfs(void **tensors, uint64_t ntypes, int dir, const uint64_t *starts, const int64_t *dests, uint64_t nstarts,
                            uint64_t min_hops, uint64_t max_hops, void **labels, uint64_t nlabels, int emit_path, uint64_t **out_p,
                            uint64_t **out_end, uint64_t **out_hops, uint64_t **path_edge, uint64_t **path_node, uint64_t *nout,
                            uint64_t *npath) {
    return var_len_c(false, tensors, ntypes, dir, starts, dests, nstarts, min_hops, max_hops, labels, nlabels, emit_path, UINT64_MAX,
                     out_p, out_end, out_hops, path_edge, path_node, nout, npath);
}

// algo.BFS (algo_bfs.hpp).  adj: the adjacency VersionedMatrix; all_types / named: Tensor pointers (nnamed = 0: no type named);
// deleted: deleted node ids; max_depth < 0 unbounded.  route 0: algo_bfs (B200_bfs_delta + B200_expand_edges); 1:
// algo_bfs_by_extract (the fresh matrix, LAGr_BreadthFirstSearch_Extended, a Tensor::get per pair).  Outputs are malloc'ed; free
// with fdbh_free.
int fdbh_algo_bfs(void *adj, void **all_types, uint64_t nall, void **named, uint64_t nnamed, const uint64_t *deleted, uint64_t ndel,
                  uint64_t src, int64_t max_depth, int want_edges, int route, uint64_t **out_nodes, uint64_t *nnodes, uint64_t **out_edges,
                  uint64_t *nedges) {
    try {
        BfsQuery q;
        q.adj = (const VersionedMatrix *)adj;
        for (uint64_t k = 0; k < nall; k++) q.all_types.push_back((const Tensor *)all_types[k]);
        for (uint64_t k = 0; k < nnamed; k++) q.named.push_back((const Tensor *)named[k]);
        if (ndel) q.deleted.assign(deleted, deleted + ndel);
        q.src = src; q.max_depth = max_depth; q.want_edges = want_edges != 0;
        if (!q.adj && q.named.empty()) throw std::invalid_argument("algo_bfs: no adjacency matrix and no type");
        BfsResult r;
        if (route == 0) r = algo_bfs(q);
        else if (route == 1) r = algo_bfs_by_extract(q);
        else throw std::invalid_argument("algo_bfs: unknown route");
        auto out = [](uint64_t **dst, const std::vector<uint64_t> &v) {
            *dst = (uint64_t *)malloc(sizeof(uint64_t) * (v.size() + 1));
            if (!*dst) throw std::bad_alloc();
            memcpy(*dst, v.data(), sizeof(uint64_t) * v.size());
        };
        out(out_nodes, r.nodes); out(out_edges, r.edges);
        *nnodes = r.nodes.size(); *nedges = r.edges.size();
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}

// shortestPath (shortest_path.hpp).  adj: the adjacency VersionedMatrix; all_types / named: Tensor pointers (nnamed = 0: no type
// named; a null entry: a named type the graph lacks); max_hops UINT64_MAX unbounded.  route 0: shortest_path (B200_shortest_path +
// B200_expand_edges); 1: shortest_path_by_iter (the reference's NeighborIter BFS and Tensor::get).  Outputs (malloc'ed; free with
// fdbh_free): p[npairs + 1] over nodes, ep[npairs + 1] over ids; a row with no node is Null.
int fdbh_shortest_path(void *adj, void **all_types, uint64_t nall, void **named, uint64_t nnamed, int directed, uint64_t min_hops,
                       uint64_t max_hops, const uint64_t *srcs, const uint64_t *dsts, uint64_t npairs, int route, uint64_t **out_p,
                       uint64_t **out_nodes, uint64_t **out_ep, uint64_t **out_ids) {
    try {
        ShortestPathQuery q;
        q.adj = (const VersionedMatrix *)adj;
        for (uint64_t k = 0; k < nall; k++) q.all_types.push_back((const Tensor *)all_types[k]);
        for (uint64_t k = 0; k < nnamed; k++) q.named.push_back((const Tensor *)named[k]);
        q.directed = directed != 0; q.min_hops = min_hops; q.max_hops = max_hops;
        if (npairs) { q.srcs.assign(srcs, srcs + npairs); q.dsts.assign(dsts, dsts + npairs); }
        ShortestPathResult r;
        if (route == 0) r = shortest_path(q);
        else if (route == 1) r = shortest_path_by_iter(q);
        else throw std::invalid_argument("shortest_path: unknown route");
        auto out = [](uint64_t **dst, const std::vector<uint64_t> &v) {
            *dst = (uint64_t *)malloc(sizeof(uint64_t) * (v.size() + 1));
            if (!*dst) throw std::bad_alloc();
            memcpy(*dst, v.data(), sizeof(uint64_t) * v.size());
        };
        out(out_p, r.p); out(out_nodes, r.nodes); out(out_ep, r.ep); out(out_ids, r.ids);
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}

// allShortestPaths (all_shortest_paths.hpp).  all_types / named: Tensor pointers (nnamed = 0: no type named; a null entry: a named
// type the graph lacks); max_hops UINT64_MAX unbounded.  route 0: all_shortest_paths (B200_all_shortest_paths, count then windows
// of at most `window` edges); 1: all_shortest_paths_by_iter (expand_row over TypesAdjacency).  Outputs (malloc'ed; free with
// fdbh_free): pp[npairs + 1] over paths, count[npairs], len[npairs], the edges and the nodes (AllShortestPathsResult's layout).
int fdbh_all_shortest_paths(void **all_types, uint64_t nall, void **named, uint64_t nnamed, int directed, uint64_t max_hops,
                            const uint64_t *srcs, const uint64_t *dsts, uint64_t npairs, int route, uint64_t window, uint64_t **out_pp,
                            uint64_t **out_count, uint64_t **out_len, uint64_t **out_edges, uint64_t **out_nodes) {
    try {
        AllShortestPathsQuery q;
        for (uint64_t k = 0; k < nall; k++) q.all_types.push_back((const Tensor *)all_types[k]);
        for (uint64_t k = 0; k < nnamed; k++) q.named.push_back((const Tensor *)named[k]);
        q.directed = directed != 0; q.max_hops = max_hops;
        if (npairs) { q.srcs.assign(srcs, srcs + npairs); q.dsts.assign(dsts, dsts + npairs); }
        AllShortestPathsResult r;
        if (route == 0) r = all_shortest_paths(q, window);
        else if (route == 1) r = all_shortest_paths_by_iter(q);
        else throw std::invalid_argument("all_shortest_paths: unknown route");
        auto out = [](uint64_t **dst, const std::vector<uint64_t> &v) {
            *dst = (uint64_t *)malloc(sizeof(uint64_t) * (v.size() + 1));
            if (!*dst) throw std::bad_alloc();
            memcpy(*dst, v.data(), sizeof(uint64_t) * v.size());
        };
        out(out_pp, r.pp); out(out_count, r.count); out(out_len, r.len); out(out_edges, r.edges); out(out_nodes, r.nodes);
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}

// algo.pageRank / algo.WCC / algo.labelPropagation (algo_procs.hpp).  adj: the adjacency VersionedMatrix; all_types / named:
// Tensor pointers (nnamed = 0: no type named; a null entry: a type the graph does not have); labels: label VersionedMatrix pointers
// (nlabels = 0: no filter; null: a missing label); node_count: live nodes; deleted: deleted node ids.  route 0: algo_proc
// (B200_adjacency_delta); 1: algo_proc_by_extract (the reference's fresh matrix).  out_nodes and out_vals (double scores or int64
// ids) are malloc'ed; free with fdbh_free.
static int algo_entry(AlgoProc proc, void *adj, void **all_types, uint64_t nall, void **named, uint64_t nnamed, void **labels,
                      uint64_t nlabels, uint64_t node_count, const uint64_t *deleted, uint64_t ndel, int max_iterations, int route,
                      uint64_t **out_nodes, void **out_vals, uint64_t *nout) {
    try {
        AlgoQuery q;
        q.proc = proc;
        q.adj = (const VersionedMatrix *)adj;
        for (uint64_t k = 0; k < nall; k++) q.all_types.push_back((const Tensor *)all_types[k]);
        for (uint64_t k = 0; k < nnamed; k++) q.named.push_back((const Tensor *)named[k]);
        for (uint64_t k = 0; k < nlabels; k++) q.labels.push_back((const VersionedMatrix *)labels[k]);
        if (ndel) q.deleted.assign(deleted, deleted + ndel);
        q.node_count = node_count;
        q.max_iterations = max_iterations;
        AlgoResult r;
        if (route == 0) r = algo_proc(q);
        else if (route == 1) r = algo_proc_by_extract(q);
        else throw std::invalid_argument("algo: unknown route");
        auto out = [](void **dst, const void *src, size_t bytes) {
            *dst = malloc(bytes + 8);
            if (!*dst) throw std::bad_alloc();
            if (bytes) memcpy(*dst, src, bytes);
        };
        out((void **)out_nodes, r.nodes.data(), 8 * r.nodes.size());
        if (proc == AlgoProc::PageRank) out(out_vals, r.score.data(), 8 * r.score.size());
        else out(out_vals, r.id.data(), 8 * r.id.size());
        *nout = r.nodes.size();
        return 0;
    } catch (const std::exception &e) { g_msg = e.what(); return 1; }
}

int fdbh_algo_pagerank(void *adj, void **all_types, uint64_t nall, void **named, uint64_t nnamed, void **labels, uint64_t nlabels,
                       uint64_t node_count, const uint64_t *deleted, uint64_t ndel, int route, uint64_t **out_nodes, double **out_score,
                       uint64_t *nout) {
    return algo_entry(AlgoProc::PageRank, adj, all_types, nall, named, nnamed, labels, nlabels, node_count, deleted, ndel, 0, route,
                      out_nodes, (void **)out_score, nout);
}

int fdbh_algo_wcc(void *adj, void **all_types, uint64_t nall, void **named, uint64_t nnamed, void **labels, uint64_t nlabels,
                  uint64_t node_count, const uint64_t *deleted, uint64_t ndel, int route, uint64_t **out_nodes, int64_t **out_id,
                  uint64_t *nout) {
    return algo_entry(AlgoProc::WCC, adj, all_types, nall, named, nnamed, labels, nlabels, node_count, deleted, ndel, 0, route,
                      out_nodes, (void **)out_id, nout);
}

int fdbh_algo_cdlp(void *adj, void **all_types, uint64_t nall, void **named, uint64_t nnamed, void **labels, uint64_t nlabels,
                   uint64_t node_count, const uint64_t *deleted, uint64_t ndel, int max_iterations, int route, uint64_t **out_nodes,
                   int64_t **out_id, uint64_t *nout) {
    return algo_entry(AlgoProc::CDLP, adj, all_types, nall, named, nnamed, labels, nlabels, node_count, deleted, ndel, max_iterations,
                      route, out_nodes, (void **)out_id, nout);
}

} // extern "C"

