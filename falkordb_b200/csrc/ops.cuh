// ops.cuh -- host-callable entry points of the kernel layer (all enqueue on b200::stream()).
#pragma once
#include "common.cuh"

namespace b200 {

// build.cu
void build_from_device_coo(const u64 *dI, const u64 *dJ, const u64 *dX, u64 n, u64 nrows, u64 ncols, DevCSR &out,
                           bool *index_error);
// GRAPH.BULK into an empty tensor: forward u64 CSR (edge id or the MULTI_EDGE sentinel) + the (pair key, id) list of multi-edge pairs
void tensor_bulk_build(const u64 *dI, const u64 *dJ, const u64 *dID, u64 n, u64 nrows, u64 ncols, DevCSR &fwd, DevBuf<u64> &mkeys,
                       DevBuf<u64> &mids, u64 *nmulti, bool *index_error);
void transpose_csr(const DevCSR &A, DevCSR &out, bool keep_values);
void rmat_csr(int scale, u64 edge_factor, u64 seed, DevCSR &out);
void rmat_block_csr(int scale, u64 edge_factor, u64 seed, u64 lo, u64 hi, int by_col, DevCSR &out);

// spgemm.cu : C = pattern(A*B) over ANY_PAIR, row-wise push (Gustavson family)
void spgemm_anypair(const DevCSR &A, const DevCSR &B, DevCSR &C, u64 *flops_out);
u64 spgemm_flops(const DevCSR &A, const DevCSR &B);

// bits.cu : the frontier bit-matrix's form, for short-fat left operands (<= 1024 rows)
u32 bits_words_for(u64 nrows);
void bits_from_csr(const DevCSR &F, DevBits &X);
void bits_to_csr(const DevBits &X, DevCSR &C);
u64 bits_nvals(const DevBits &X);
void bits_naturalise(DevBits &X);                                // permuted form -> natural vertex order (no-op when natural)
bool csr_is_diagonal(const DevCSR &A);                          // square, every entry (i,i)
void bits_diag(const DevBits &X, const DevCSR &A, DevBits &Y, u64 *flops_out);   // Y = X * A for diagonal A
void bits_to_rowmajor(const DevBits &X, u64 *out, u64 wpr);   // out[row * wpr + (col >> 6)], every word written
void csr_to_rowmajor(const DevCSR &A, u64 *out, u64 wpr);     // out must be zero on entry
void bits_andnot(DevBits &Y, const DevBits &M); // Y &= ~M
void bits_or(DevBits &Y, const DevBits &Z);     // Y |= Z
void bits_copy(const DevBits &X, DevBits &Y);

struct PullTables;
// csr_push.cu : the push straight from a CSR frontier, and the delta terms of delta_lmxm
// Y = F * A expanded straight from F's CSR (small frontiers); false = the frontier touches enough of A that the pull should take
// it (edges * 4 > nnz(A)), nothing was done.  pt (optional): A's pull tables; when they carry a vertex order the result is
// written in it (permuted form).  acc: Y |= F * A, Y holding a natural-order product of the same shape (pt is then ignored)
bool bits_push_from_csr(const DevCSR &F, const DevCSR &A, DevBits &Y, u64 *flops_out, const PullTables *pt = nullptr,
                        bool acc = false);
// The delta terms of delta_lmxm applied in place to Y = X * m:  Y = (Y AND NOT X * dm) OR X * dp, one pass over each delta's
// entries.  The left operand is the bit-matrix Xb, or the CSR Xc when Y came from bits_push_from_csr (Xb null).  dm / dp may be
// null.  X and Y stay in the vertex order they are stored in.  Returns flops(X * dm) + flops(X * dp).
u64 bits_apply_deltas(const DevBits *Xb, const DevCSR *Xc, const DevCSR *dm, const DevCSR *dp, DevBits &Y);

// bits_hop.cu : the bit-matrix hop (push or pull) and the exact dirty-hop repair
struct PullTables {   // per-matrix tables of the pull direction, cached with the transpose mirror
    // hot-set order: vertices with out-edges, by out-degree descending
    DevBuf<u32> vert, slot, hdeg; u64 n1 = 0; bool packed = false;   // hdeg[s] = out-degree of vert[s]
    // the same order extended to ALL vertices (sinks follow the n1 slots, by id): a frontier stored in it needs no packing pass
    std::shared_ptr<DevBuf<u32>> pvert, pperm; u64 perm_tag = 0;    // pvert[position] = vertex, pperm[vertex] = position
    DevBuf<u32> jp;                                    // col_idx of A' relabelled to hot-set slots (when packed)
    DevBuf<u32> ap;                                    // col_idx of A relabelled to positions (pperm[A.j], when packed): the CSR push's operand
    bool ap_sorted = false;                            // every row of ap ascending by position: the push may cut it into destination slices
    // segment list: rows of A' longer than SMALL_ROW -- whole rows up to LONG_ROW entries, LONG_ROW-entry segments of longer ones --
    // longest first; bit 31 of s_len marks a segment of a long row (merged with RED.OR)
    DevBuf<u32> s_row, s_len; DevBuf<u64> s_start; u64 ns = 0;
    bool built = false;                                // the segment list is built
    void clear() {
        vert.release(); slot.release(); hdeg.release(); n1 = 0; packed = false; pvert.reset(); pperm.reset(); perm_tag = 0;
        jp.release(); ap.release(); ap_sorted = false;
        s_row.release(); s_len.release(); s_start.release(); ns = 0;
        built = false;
    }
};
// Y = X * A.  AT (= A') and its pull tables enable the pull direction; may be null (push only).  acc: Y |= X * A into a
// natural-order Y of the product's shape (the push skips zeroing Y, the pull ORs each row into the stored record).
void bits_hop(const DevBits &X, const DevCSR &A, const DevCSR *AT, PullTables *pt, DevBits &Y, u64 *flops_out,
              int *path_out, bool acc = false);
void bits_prepare_pull(const DevCSR &A, const DevCSR &AT, PullTables &pt);   // square A: build the pull tables now
// The exact dirty hop's deleted-edge term.  For every column j that dm touches, Y[j] = OR of X[k] over the in-edges k of m(:, j)
// that are not in dm (Y = X * (m \ dm) on those columns; every other column of X * m is already exact).  The plan is built once
// per operand and call: dmT = dm', and the repaired columns of m' (m's transpose mirror, natural column ids) cut into segments of
// at most REPAIR_SEG in-edges; a column of several segments is zeroed and its segments merged with RED.OR.
struct RepairPlan {
    DevCSR dmT;                                        // row j = the deleted sources of column j, ascending
    DevBuf<u32> s_col, s_len; DevBuf<u64> s_start;     // segment -> column, length | flags, first position in m'.col_idx
    u64 ns = 0, ncols = 0, inedges = 0;                // segments, repaired columns, in-edges of m over them
};
void bits_repair_plan(const DevCSR &dm, const DevCSR &mT, RepairPlan &rp);
void bits_repair(const DevBits &X, const DevCSR &mT, const RepairPlan &rp, DevBits &Y);

// ewise.cu : search-based set algebra on sorted CSR rows
void csr_copy(const DevCSR &A, DevCSR &out, bool keep_values);
void ewise_union(const DevCSR &A, const DevCSR &B, bool keep_values, DevCSR &out); // overlap: B's value (SECOND)
void ewise_intersect(const DevCSR &A, const DevCSR &B, DevCSR &out);               // pattern only
// keep t in T iff (t in M [and M's value != 0 unless structural]) XOR comp
void filter_by_mask(const DevCSR &T, const DevCSR &M, bool comp, bool structural, DevCSR &out);
void csr_resize(const DevCSR &A, u64 nrows, u64 ncols, DevCSR &out); // grow/shrink dims (drops out-of-range)
// Z = pattern(A*B) restricted to M's structure (valued mask: entries of M with value 0 excluded unless structural)
void spgemm_masked(const DevCSR &A, const DevCSR &B, const DevCSR &M, bool structural, DevCSR &out, u64 flops = 0);

void csr_digest(const DevCSR &A, u64 *host_out3);   // {nnz, sum mix(key), sum mix(key + GOLD * (pos + 1))}: see oracle orc_digest
// bfs_do.cu : direction-optimising BFS, single GPU or 1-D row-block partitioned over NCCL; top-down BFS without A'
struct BfsComm;
struct BfsInfo {          // mirrored by B200_BfsInfo in include/b200grb.h
    u64 depth, edges, td_levels, bu_levels, sparse_levels, exchanges, exchanged_bytes;
    double device_ms, exchange_ms;
};
void comm_unique_id(unsigned char *id128);
BfsComm *comm_init(int rank, int world, const unsigned char *id128);
void comm_free(BfsComm *c);
int comm_rank(const BfsComm *c);
int comm_world(const BfsComm *c);
void comm_allgather(BfsComm *c, const void *send, void *recv, size_t bytes_per_rank);
void bfs_build_degrees(const DevCSR &Aloc, u64 n, u64 lo, u64 hi, BfsComm *comm, DevBuf<u32> &deg_all, u64 *total_edges);
// one operand of the BFS over A = U_t (m_t \ dm_t) u dp_t: the base, its transpose mirror and its cached out-degree table (edges =
// nnz(m)); dp and dm and their per-call transposes (null: empty)
struct BfsOperand {
    const DevCSR *m, *mT, *dp, *dpT, *dm, *dmT;
    const u32 *deg; u64 edges;
};
void bfs_delta_degrees(const std::vector<BfsOperand> &ops, u64 n, DevBuf<u32> &deg, u64 *total_edges);   // the switch's table
// dirty (one GPU): the operands A is the union of; Aloc / ATloc are then not read, deg_all / total_edges from bfs_delta_degrees
void bfs_do(const DevCSR &Aloc, const DevCSR &ATloc, u64 n, u64 lo, u64 hi, const u32 *deg_all, u64 total_edges, BfsComm *comm,
            u64 src, i64 max_level, i64 dest, i64 *d_level, i64 *d_parent, BfsInfo *info,
            const std::vector<BfsOperand> *dirty = nullptr);
void bfs_run(const DevCSR &A, u64 src, i64 max_level, i64 *d_level, i64 *d_parent, u64 *edges_traversed);

// algo.cu : FP64 mxv (PLUS_TIMES / PLUS_SECOND) and PageRank
void mxv_fp64(const DevCSR &A, bool use_values, const double *x, const unsigned char *present, double *y, unsigned char *ypresent,
              double init, bool accum);
int pagerank(const DevCSR &A, const DevCSR &AT, double damping, double tol, int itermax, double *r);
int connected_components(const DevCSR &A, u64 *d_comp);     // symmetric pattern; d_comp[v] = smallest vertex id of v's component
int cdlp(const DevCSR &A, int itermax, u64 *d_label);         // synchronous label propagation, min label on ties; returns the rounds run

void probe_pairs(const DevCSR &A, const u64 *dI, const u64 *dJ, u64 n, unsigned char *d_found, u64 *d_val);

// edges.cu : relationship ids of the rows of a batch over relationship tensors' live layers (B200_expand_edges)
struct DevIdStore {   // a host-resident matrix's sorted store on the device: key[k] = a non-empty row, its columns id[ptr[k] .. ptr[k+1])
    DevBuf<u64> key, ptr, id;
    u64 nkey = 0;
    bool valid = false;
    void upload(const u64 *hkey, const u64 *hptr, const u64 *hid, u64 nk);
    void clear() { key.release(); ptr.release(); id.release(); nkey = 0; valid = false; }
};
struct EdgeTypeDev {  // one relationship type: forward m / dp (u64 values) / dm, the transpose's layers, the multi-edge store's
    const DevCSR *m, *dp, *dm, *mt, *mt_dp, *mt_dm;   // null or empty: absent
    const DevIdStore *me, *me_dp, *me_dm;
};
// dir 0 out / 1 in / 2 both, mode 0 every id / 1 the first id per (row, block, neighbour).  d_tgt null: every neighbour.  Writes
// out_p[0..n] and returns the number of output entries; the entries themselves only when they fit in capacity.
u64 edge_expand(const u64 *d_src, const u64 *d_tgt, u64 n, const std::vector<EdgeTypeDev> &types, int dir, int mode, u64 *out_p,
                u32 *out_node, u64 *out_edge, uint16_t *out_type, uint8_t *out_rev, u64 capacity);

// writes.cu : the read phase of a Tensor's batched relationship inserts and deletes (B200_Tensor_insert_plan / _remove_plan),
// over one type's live layers (m, dp, dm, mt and the me stores of EdgeTypeDev; mt_dp / mt_dm are not read).  The flags are
// include/b200grb.h's B200_PLAN_*.  The plan goes to the caller's host arrays: rec_* (capacity n) and me_* (capacity 2n).
enum : uint8_t { WP_COMMITTED = 1, WP_CANCEL = 2, WP_MT_BASE = 4, WP_EMPTIED = 8, WP_DEMOTED = 16, WP_M_HAS = 32, WP_M_EQ = 64 };
struct WritePlan {
    u64 *rec_src, *rec_dst, *rec_val; uint8_t *rec_flags; u64 nrec;
    u64 *me_key, *me_id; uint8_t *me_base; u64 nme;
};
// n >= 1; src / dst < nv, ids < 2^60 (checked by the caller)
void tensor_insert_plan(const EdgeTypeDev &t, const u64 *d_src, const u64 *d_dst, const u64 *d_id, u64 n, u64 nv, WritePlan &P);
void tensor_remove_plan(const EdgeTypeDev &t, const u64 *d_id, const u64 *d_src, const u64 *d_dst, u64 n, u64 nv, WritePlan &P);

// trails.cu : CondVarLenTraverse's trails for a batch of starts (B200_var_len_trails) over relationship tensors' live layers
struct LabelDev { const DevCSR *m, *dp, *dm; };   // one destination label's layers (null or empty: absent)
struct TrailsOut {
    u64 *out_p;                                    // host, nstarts + 1
    u32 *out_end, *out_hops;                       // host; out_end null: count only
    u64 *path_edge; u32 *path_node;                // host; path_edge null: no paths
    u64 out_capacity, path_capacity;
    u64 nout = 0, npath = 0;
};
// nstarts >= 1, starts < nv and min_hops <= max_hops (checked by the caller); dir 0 out / 1 in / 2 both; h_dests null or < 0: no
// fixed destination.  Returns 0 (done), 1 (the outputs do not fit: only out_p, nout and npath written) or 2 (the stored trail tree
// would exceed tree_capacity entries: nothing written).
int var_len_trails(const u64 *h_starts, const i64 *h_dests, u64 nstarts, const std::vector<EdgeTypeDev> &types, int dir, u64 min_hops,
                   u64 max_hops, const std::vector<LabelDev> &labels, u64 nv, u64 tree_capacity, TrailsOut &o);

// var_len_reach.cu : whether a bidirectional variable-length reach (B200_var_len_reach_both) emits each start itself, i.e. whether
// the undirected multigraph of the types holds a cycle through it of at most max_hops edges
struct VlbPlan {
    u64 n = 0, nu = 0, Q = 0, rows = 0;           // starts, distinct starts, their distinct neighbours other than themselves, closure rows
    DevBuf<u64> ds, u;                             // the starts; the distinct starts, ascending
    DevBuf<u32> slot, dec;                         // per start its slot in u; per slot 1 = the start is emitted
    DevBuf<u32> dn, dslot;                         // the distinct neighbours, slot-major, ascending within a slot
    DevBuf<u64> nbase, rowbase;                    // per slot (nu + 1): its first distinct neighbour, its first closure row
    u64 q0 = 0, q1 = 0;                            // the current chunk's distinct neighbours
};
// nstarts >= 1, starts < nv (checked by the caller); the short cycles (g <= 2) decided, the rows of the longer ones laid out
void vlb_plan(const u64 *h_starts, u64 nstarts, const std::vector<EdgeTypeDev> &types, u64 max_hops, VlbPlan &P);
// closure rows [r0, r1) (at most 1024): F = the seeds, R = the seeds and the start, W = bits_words_for(r1 - r0)
void vlb_seed(VlbPlan &P, u64 r0, u64 r1, u64 n, DevBits &F, DevBits &R);
// after a level of F: rows whose frontier meets their targets decide their start; every row of a decided start leaves F.
// Returns the rows with a frontier left.
u64 vlb_level(VlbPlan &P, u64 r0, u64 r1, DevBits &F);
// (i, starts[i]) cleared in row i of the reach unless the start is emitted: the bit-matrix in place, or a CSR into out
void vlb_fix_bits(const VlbPlan &P, DevBits &R);
void vlb_fix_csr(const VlbPlan &P, const DevCSR &R, DevCSR &out);

// shortest_path.cu : shortestPath's bidirectional BFS (B200_shortest_path) for np pairs with src != dst (< n, checked by the caller).
// Each side is a union of operands (m \ dm) u dp, pattern only.  len[i] = nodes on pair i's path (0: Null); nodes = the paths,
// concatenated, from src to dst.  budget: neighbour entries per piece of a round (0: from free memory).  Returns the neighbour
// entries scanned.
struct SpOperand { const DevCSR *m, *dp, *dm; };
u64 shortest_path(const u64 *h_src, const u64 *h_dst, u64 np, const std::vector<SpOperand> &fwd, const std::vector<SpOperand> &bwd,
                  u64 n, u64 max_hops, u64 budget, std::vector<u64> &len, std::vector<u32> &nodes);

// all_shortest_paths.cu : allShortestPaths' every shortest path (B200_all_shortest_paths) for np >= 1 pairs (< n and max_hops >= 1,
// checked by the caller) over relationship types' live layers (every type with its transpose), dir 0 out / 2 both.  Per pair:
// count (saturating), len (edges per path, 0 when none), out_p (np + 1, paths written, a prefix); path_edge null: count only,
// else from rank h_first[i] (null: 0) on, pair after pair, until a path no longer fits edge_capacity.  budget: candidates per
// piece of a forward level (0: from free memory).  Returns the adjacency entries scanned.
u64 all_shortest_paths(const u64 *h_src, const u64 *h_dst, u64 np, const std::vector<EdgeTypeDev> &types, int dir, u64 n,
                       u64 max_hops, u64 budget, const u64 *h_first, u64 *count, u32 *len, u64 *out_p, u64 *path_edge,
                       u32 *path_node, u64 edge_capacity, u64 *nedges);

// adj.cu : the induced effective layer (B200_adjacency_delta).  out = L \ dm restricted to kept rows and columns, both indices
// replaced by their rank: d_keep null, rank(v) = v below n_out (out is n_out x n_out); else d_keep[0 .. nkeep) strictly ascending
// and rank_tab from adj_rank_table (out is nkeep x nkeep).  dm may be null.  Pattern only.
void adj_rank_table(const u64 *d_keep, u64 nkeep, u64 n, DevBuf<u32> &tab);   // tab[v] = v's position in keep, or ~0u
void adj_layer(const DevCSR &L, const DevCSR *dm, u64 n_out, const u64 *d_keep, const u32 *rank_tab, u64 nkeep, DevCSR &out);

// hypersparse host form <-> dense device rowptr (ewise.cu)
void rowptr_from_hyper(const u64 *d_hrow, const u64 *d_hptr, u64 nvec, u64 nrows, u64 *d_p);
u64 hyper_from_rowptr(const u64 *d_p, u64 nrows, u64 nnz, DevBuf<u64> &d_hrow, DevBuf<u64> &d_hptr);

} // namespace b200
