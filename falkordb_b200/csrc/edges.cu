// edges.cu -- relationship ids of named-edge, incoming and bidirectional hops (B200_expand_edges): the edges CondTraverse's
// expand_row / bind_edge and ExpandInto read one Tensor::get at a time (cond_traverse.rs:663-702, 844-935, expand_into.rs:121-258),
// for a whole batch of rows in one pass over the tensors' live layers.
//
// Lists.  Row i, block b (forward: out-neighbours; reverse: in-neighbours), type t and layer l (0 = the base m / mt, 1 = the
// delta-plus dp / mt_dp) own one list: the layer's row sources[i], or with targets only its entry at targets[i] (0 or 1 entry).
// Lists are laid out flat in (row, block, type, layer) order behind an exclusive scan of their lengths, and every pass runs one
// thread per list entry, so a hub row is spread over the whole grid like any other.
// Count.  A base entry shadowed by its delta-minus or delta-plus layer counts 0.  A forward entry's value is its layer value; a
// reverse entry (k in row s of mt) looks its value up at forward (k, s) with Tensor::eff_get's rule.  The count is 1, or for a
// MULTI_EDGE value the size of the key's merged id list (me \ me_dm) u me_dp.  EDGES_FIRST keeps 1 for the first type present
// at a neighbour and 0 for the others.
// Place.  Lists are sorted by neighbour, so an entry's output position is the block's offset plus, per list of its block, the
// counts of the entries ahead of it -- smaller neighbours, and the same neighbour in a lower-index type -- read from the scan of
// the counts with one binary search per list (2T per entry; ewise.cu's rank sums).  No sort and no merge loop.
// Fill.  node, id, type and direction of every output entry; a MULTI_EDGE entry writes its merged id list.
// edge_adjacency (the trail enumerator's per-level fetch, trails.cu) runs the same lists, counts and scan over device-resident
// rows, and places the entries in Graph::get_node_relationships_by_type's order instead (k_ee_ref_fill): type, block, neighbour.
// The me layers are host-resident (2^60 x 2^60); their sorted (key, ids) stores are uploaded once and cached on the handle.
#include "edge_layers.cuh"
#include <type_traits>

namespace b200 {

struct EArgs {
    const u64 *src, *tgt;            // tgt null: every neighbour
    const EType *types;
    u64 n, G, E;                     // rows, lists, list entries
    u32 T, nb;                       // types, blocks per row
    int dir;
};

struct ListId { u64 i; u32 b, t, l; bool rev; };
__device__ __forceinline__ ListId list_of(const EArgs &A, u64 g) {
    ListId r;
    r.l = (u32)(g & 1);
    u64 q = g >> 1;
    r.t = (u32)(q % A.T); q /= A.T;
    r.b = (u32)(q % A.nb);
    r.i = q / A.nb;
    r.rev = A.dir == 1 || (A.dir == 2 && r.b == 1);
    return r;
}
__device__ __forceinline__ const ECsr &layer_of(const EType &t, bool rev, u32 l) { return rev ? (l ? t.mtdp : t.mt) : (l ? t.dp : t.m); }

// per list: its first position in the layer's col_idx and its length.  stat[0] += forward entries, stat[1] += reverse entries,
// stat[2] += entries of the delta-minus rows the count pass searches (the byte formula)
__global__ void k_ee_lists(EArgs A, u64 *__restrict__ lo, u64 *__restrict__ len, u64 *__restrict__ stat) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < A.G; g += (u64)gridDim.x * blockDim.x) {
        const ListId L = list_of(A, g);
        const EType &t = A.types[L.t];
        const ECsr &X = layer_of(t, L.rev, L.l);
        const u64 s = A.src[L.i];
        u64 a = 0, n = 0;
        if (X.p) {
            a = X.p[s];
            u64 e = X.p[s + 1];
            if (A.tgt) { const u32 c = (u32)A.tgt[L.i]; a = lb32(X.j, a, e, c); e = a < e && X.j[a] == c ? a + 1 : a; }
            n = e - a;
        }
        lo[g] = a; len[g] = n;
        if (n) atomicAdd((unsigned long long *)&stat[L.rev ? 1 : 0], (unsigned long long)n);
        const ECsr &D = L.rev ? t.mtdm : t.dm;
        if (L.l == 0 && D.p && D.p[s + 1] > D.p[s]) atomicAdd((unsigned long long *)&stat[2], (unsigned long long)(D.p[s + 1] - D.p[s]));
    }
}

// per entry: value and count (ALL semantics)
__global__ void k_ee_count(EArgs A, const u64 *__restrict__ lstart, const u64 *__restrict__ lo, u64 *__restrict__ val,
                           u32 *__restrict__ cnt) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < A.E; e += (u64)gridDim.x * blockDim.x) {
        const u64 g = list_at(lstart, A.G, e);
        const ListId L = list_of(A, g);
        const EType &t = A.types[L.t];
        const ECsr &X = layer_of(t, L.rev, L.l);
        const u64 s = A.src[L.i], q = lo[g] + (e - lstart[g]);
        const u32 x = X.j[q];
        u32 c = 0;
        u64 v = 0;
        bool live = !(A.dir == 2 && L.rev && x == s);                         // BOTH: a self-loop once, in the forward block
        if (live && L.l == 0)                                                  // a base entry the deltas shadow
            live = find_rc(L.rev ? t.mtdm : t.dm, s, x) == ~0ULL && find_rc(L.rev ? t.mtdp : t.dp, s, x) == ~0ULL;
        if (live) {
            if (!L.rev) v = X.x[q];
            else live = eff_get(t, x, (u32)s, &v);                             // in-neighbour x: the forward pair (x, s)
        }
        if (live) {
            if (v != EE_MULTI) c = 1;
            else {
                const u64 key = L.rev ? ((u64)x << 32 | s) : (s << 32 | x);
                c = (u32)merged_ids(t, key, [](u64, u64) { return true; });
            }
        }
        val[e] = v; cnt[e] = c;
    }
}

// entry e of list g: where neighbour x sits in list g2 of the same block -- the entries ahead of it (< x, or <= x for a
// lower-index type) as a flat position
__device__ __forceinline__ u64 rank_in(const EArgs &A, const u64 *__restrict__ lstart, const u64 *__restrict__ lo,
                                       const u64 *__restrict__ len, u64 g2, bool rev, u32 x, bool upper) {
    const ListId L2 = list_of(A, g2);
    const ECsr &X = layer_of(A.types[L2.t], rev, L2.l);
    const u64 a = lo[g2], b = a + len[g2];
    if (a == b) return lstart[g2];
    const u64 k = upper ? ub32(X.j, a, b, x) : lb32(X.j, a, b, x);
    return lstart[g2] + (k - a);
}

// EDGES_FIRST: an entry keeps 1 when no lower-index type of its block holds a counted entry at the same neighbour
__global__ void k_ee_first(EArgs A, const u64 *__restrict__ lstart, const u64 *__restrict__ lo, const u64 *__restrict__ len,
                           const u32 *__restrict__ cnt, u32 *__restrict__ first) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < A.E; e += (u64)gridDim.x * blockDim.x) {
        u32 keep = 0;
        if (cnt[e]) {
            const u64 g = list_at(lstart, A.G, e);
            const ListId L = list_of(A, g);
            const u32 x = layer_of(A.types[L.t], L.rev, L.l).j[lo[g] + (e - lstart[g])];
            const u64 blk = g - (g % (2 * (u64)A.T));
            keep = 1;
            for (u32 t2 = 0; t2 < L.t && keep; t2++)
                for (u32 l2 = 0; l2 < 2; l2++) {
                    const u64 g2 = blk + 2 * t2 + l2;
                    const u64 e2 = rank_in(A, lstart, lo, len, g2, L.rev, x, false);
                    const ListId M = list_of(A, g2);
                    const ECsr &X = layer_of(A.types[M.t], L.rev, M.l);
                    if (e2 < lstart[g2] + len[g2] && X.j[lo[g2] + (e2 - lstart[g2])] == x && cnt[e2]) { keep = 0; break; }
                }
        }
        first[e] = keep;
    }
}

// out_p[i] = the output position of row i's first list (i = n: the total)
__global__ void k_ee_rowptr(EArgs A, const u64 *__restrict__ lstart, const u64 *__restrict__ pos, u64 *__restrict__ out_p) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= A.n; i += (u64)gridDim.x * blockDim.x)
        out_p[i] = pos[lstart[i * A.nb * 2 * A.T]];
}

__global__ void k_ee_fill(EArgs A, const u64 *__restrict__ lstart, const u64 *__restrict__ lo, const u64 *__restrict__ len,
                          const u64 *__restrict__ val, const u32 *__restrict__ cnt, const u64 *__restrict__ pos,
                          u32 *__restrict__ node, u64 *__restrict__ edge, uint16_t *__restrict__ type, uint8_t *__restrict__ rev) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < A.E; e += (u64)gridDim.x * blockDim.x) {
        const u32 c = cnt[e];
        if (!c) continue;
        const u64 g = list_at(lstart, A.G, e);
        const ListId L = list_of(A, g);
        const EType &t = A.types[L.t];
        const u32 x = layer_of(t, L.rev, L.l).j[lo[g] + (e - lstart[g])];
        const u64 blk = g - (g % (2 * (u64)A.T));
        u64 o = pos[lstart[blk]];                                              // row offset + the blocks before this one
        for (u32 t2 = 0; t2 < A.T; t2++)
            for (u32 l2 = 0; l2 < 2; l2++) {
                const u64 g2 = blk + 2 * t2 + l2;
                const u64 e2 = g2 == g ? e : rank_in(A, lstart, lo, len, g2, L.rev, x, t2 < L.t);
                o += pos[e2] - pos[lstart[g2]];
            }
        const u64 v = val[e];
        auto put = [&](u64 k, u64 id) {
            node[o + k] = x;
            edge[o + k] = id;
            if (type) type[o + k] = (uint16_t)L.t;
            if (rev) rev[o + k] = L.rev ? 1 : 0;
            return k + 1 < c;
        };
        if (v != EE_MULTI) put(0, v);
        else {
            const u64 s = A.src[L.i];
            merged_ids(t, L.rev ? ((u64)x << 32 | s) : (s << 32 | x), put);
        }
    }
}

// The reference's order (edge_adjacency): per row, type, then block (outgoing, then incoming), then neighbour and id.  An entry's
// position is the row offset, plus the counts of every list of an earlier (type, block), plus the entries ahead of it in its own
// list and in the other layer of its (type, block) -- one binary search.  A base entry and a delta-plus entry never both count.
__global__ void k_ee_ref_fill(EArgs A, const u64 *__restrict__ lstart, const u64 *__restrict__ lo, const u64 *__restrict__ len,
                              const u64 *__restrict__ val, const u32 *__restrict__ cnt, const u64 *__restrict__ pos,
                              u32 *__restrict__ node, u64 *__restrict__ edge, u32 *__restrict__ tb) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < A.E; e += (u64)gridDim.x * blockDim.x) {
        const u32 c = cnt[e];
        if (!c) continue;
        const u64 g = list_at(lstart, A.G, e);
        const ListId L = list_of(A, g);
        const EType &t = A.types[L.t];
        const u32 x = layer_of(t, L.rev, L.l).j[lo[g] + (e - lstart[g])];
        const u64 row = g - (g % (2 * (u64)A.T * A.nb));
        u64 o = pos[lstart[row]];
        for (u32 t2 = 0; t2 <= L.t; t2++)
            for (u32 b2 = 0; b2 < A.nb && (t2 < L.t || b2 < L.b); b2++) {
                const u64 g2 = row + 2 * ((u64)b2 * A.T + t2);
                o += pos[lstart[g2 + 2]] - pos[lstart[g2]];
            }
        const u64 g0 = g & ~1ULL;
        for (u32 l2 = 0; l2 < 2; l2++) {
            const u64 g2 = g0 + l2;
            const u64 e2 = g2 == g ? e : rank_in(A, lstart, lo, len, g2, L.rev, x, false);
            o += pos[e2] - pos[lstart[g2]];
        }
        const u64 v = val[e];
        auto put = [&](u64 k, u64 id) {
            node[o + k] = x;
            edge[o + k] = id;
            if (tb) tb[o + k] = L.t << 1 | (L.rev ? 1 : 0);
            return k + 1 < c;
        };
        if (v != EE_MULTI) put(0, v);
        else {
            const u64 s = A.src[L.i];
            merged_ids(t, L.rev ? ((u64)x << 32 | s) : (s << 32 | x), put);
        }
    }
}

// The passes before the fill, shared by both orders: the lists, their entries' values and counts, and the scan of the counts.
struct EeBatch {
    EArgs A;
    DevBuf<u64> lo, llen, lstart, stat, val, pos;
    DevBuf<u32> cnt, first;
    u32 *fin = nullptr;
    u64 h[4] = {0, 0, 0, 0};         // forward entries, reverse entries, delta-minus entries searched, list entries
    explicit EeBatch(const EArgs &a) : A(a), lo(a.G), llen(a.G + 1), lstart(a.G + 1), stat(3) { stat.zero(); }
    void prepare(int mode, u32 grid) {
        CUDA_TRY(cudaMemsetAsync(llen.ptr + A.G, 0, sizeof(u64), stream()));
        LAUNCH(k_ee_lists, grid_for(A.G, 256, grid), 256, 0, A, lo.ptr, llen.ptr, stat.ptr);
        exclusive_scan_u64(llen.ptr, lstart.ptr, A.G + 1);
        d2h(h, stat.ptr, 3);
        d2h(h + 3, lstart.ptr + A.G, 1);
        sync_stream();
        A.E = h[3];
        val.alloc(A.E); pos.alloc(A.E + 1); cnt.alloc(A.E + 1);
        fin = cnt.ptr;
        CUDA_TRY(cudaMemsetAsync(cnt.ptr + A.E, 0, sizeof(u32), stream()));
        if (A.E) LAUNCH(k_ee_count, grid_for(A.E, 256, grid), 256, 0, A, lstart.ptr, lo.ptr, val.ptr, cnt.ptr);
        if (mode == 1 && A.E) {
            first.alloc(A.E + 1);
            CUDA_TRY(cudaMemsetAsync(first.ptr + A.E, 0, sizeof(u32), stream()));
            LAUNCH(k_ee_first, grid_for(A.E, 256, grid), 256, 0, A, lstart.ptr, lo.ptr, llen.ptr, cnt.ptr, first.ptr);
            fin = first.ptr;
        }
        exclusive_scan_u32_to_u64(fin, pos.ptr, A.E + 1);
    }
    u64 bytes() const { return 16 * A.G + 12 * h[0] + 28 * h[1] + 4 * h[2]; }
};

ETypes::ETypes(const std::vector<EdgeTypeDev> &types) : d(types.size()), T((u32)types.size()) {
    std::vector<EType> h(T);
    for (u32 t = 0; t < T; t++) h[t] = etype(types[t]);
    h2d(d.ptr, h.data(), T);
}

u64 edge_adjacency(const ETypes &types, const u64 *d_src, u64 n, int dir, DevBuf<u64> &p, DevBuf<u32> &node, DevBuf<u64> &edge,
                   u64 *bytes, DevBuf<u32> *tb) {
    const u32 T = types.T, nb = dir == 2 ? 2 : 1, grid = (u32)ctx().num_sms * 8;
    EeBatch B(EArgs{d_src, nullptr, types.d.ptr, n, n * nb * T * 2, 0, T, nb, dir});
    B.prepare(0, grid);
    p.alloc(n + 1);
    LAUNCH(k_ee_rowptr, grid_for(n + 1, 256, grid), 256, 0, B.A, B.lstart.ptr, B.pos.ptr, p.ptr);
    u64 total = 0;
    d2h(&total, p.ptr + n, 1);
    sync_stream();
    node.alloc(total); edge.alloc(total);
    if (tb) tb->alloc(total);
    if (total)
        LAUNCH(k_ee_ref_fill, grid_for(B.A.E, 256, grid), 256, 0, B.A, B.lstart.ptr, B.lo.ptr, B.llen.ptr, B.val.ptr, B.fin, B.pos.ptr,
               node.ptr, edge.ptr, tb ? tb->ptr : nullptr);
    *bytes += B.bytes() + (tb ? 16 : 12) * total;
    return total;
}

__global__ void k_adj_low(const u64 *__restrict__ key, u64 n, u64 *__restrict__ out) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) out[i] = (u32)key[i];
}
template <class K>
__global__ void k_adj_rows(const K *__restrict__ key, u64 n, const u64 *__restrict__ u, u64 nu, const u64 *__restrict__ adj_p,
                           u32 *__restrict__ row, u64 *__restrict__ deg) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (u64)gridDim.x * blockDim.x) {
        u64 d = 0;
        if (i < n) {
            const u64 a = lb64(u, 0, nu, (u32)key[i]);
            row[i] = (u32)a;
            if (deg) d = adj_p[a + 1] - adj_p[a];
        }
        if (deg) deg[i] = d;
    }
}
template <class K>
void node_rows(const K *keys, u64 n, const u64 *u, u64 nu, const u64 *adj_p, u32 *row, u64 *deg) {
    LAUNCH(k_adj_rows<K>, grid_for(n + 1, 256), 256, 0, keys, n, u, nu, adj_p, row, deg);
}
template <class K>
void NodeAdj::fetch(const ETypes &types, const K *keys, u64 n, int dir, bool want_tb, u64 *bytes) {
    u.alloc(n);
    if constexpr (std::is_same<K, u32>::value) widen_u32(keys, u.ptr, n);
    else LAUNCH(k_adj_low, grid_for(n, 256), 256, 0, keys, n, u.ptr);
    const u64 nu = unique_sorted(u, n, 32);
    edge_adjacency(types, u.ptr, nu, dir, p, node, edge, bytes, want_tb ? &tb : nullptr);
    row.alloc(n);
    cum.alloc(n + 1);
    node_rows(keys, n, u.ptr, nu, p.ptr, row.ptr, cum.ptr);
    exclusive_scan_u64(cum.ptr, cum.ptr, n + 1);
    total = read_scalar(cum.ptr + n);
}
template void node_rows<u64>(const u64 *, u64, const u64 *, u64, const u64 *, u32 *, u64 *);
template void NodeAdj::fetch<u32>(const ETypes &, const u32 *, u64, int, bool, u64 *);
template void NodeAdj::fetch<u64>(const ETypes &, const u64 *, u64, int, bool, u64 *);

// the end of the piece starting at front entry i0: the last i1 with cum[i1] - cum[i0] <= budget, at least i0 + 1
__global__ void k_piece_cut(const u64 *__restrict__ cum, u64 i0, u64 nf, u64 budget, u64 *__restrict__ out) {
    u64 a = i0 + 1, b = nf;
    while (a < b) { u64 mid = (a + b + 1) >> 1; if (cum[mid] - cum[i0] <= budget) a = mid; else b = mid - 1; }
    *out = a;
}
void for_each_piece(const u64 *cum, u64 nf, u64 total, u64 budget, const std::function<void(u64, u64, u64, u64)> &f) {
    DevBuf<u64> end(1);
    for (u64 i0 = 0, q0 = 0; q0 < total;) {
        u64 i1 = nf;
        if (total - q0 > budget) {
            LAUNCH(k_piece_cut, 1, 1, 0, cum, i0, nf, budget, end.ptr);
            i1 = read_scalar(end.ptr);
        }
        const u64 q1 = i1 < nf ? read_scalar(cum + i1) : total;
        if (q1 > q0) f(i0, i1, q0, q1);
        i0 = i1; q0 = q1;
    }
}

void for_each_slice(u64 np, u64 S_max, const std::function<void(u64, u64)> &run_slice) {
    u64 S_cur = S_max;
    for (u64 p0 = 0; p0 < np;) {
        const u64 S = std::min<u64>(S_cur, np - p0);
        try {
            run_slice(p0, S);
        } catch (const CudaError &e) {
            if (e.code != cudaErrorMemoryAllocation || S == 1) throw;
            cudaGetLastError();
            pool_trim();
            S_cur = S / 2;
            continue;
        }
        p0 += S;
    }
}

void DevIdStore::upload(const u64 *hkey, const u64 *hptr, const u64 *hid, u64 nk) {
    clear();
    nkey = nk;
    if (nk) {
        key.alloc(nk); ptr.alloc(nk + 1); id.alloc(hptr[nk]);
        h2d(key.ptr, hkey, nk); h2d(ptr.ptr, hptr, nk + 1); h2d(id.ptr, hid, hptr[nk]);
        sync_stream();                                   // the host vectors are pageable
    }
    valid = true;
}

u64 edge_expand(const u64 *d_src, const u64 *d_tgt, u64 n, const std::vector<EdgeTypeDev> &types, int dir, int mode, u64 *out_p,
                u32 *out_node, u64 *out_edge, uint16_t *out_type, uint8_t *out_rev, u64 capacity) {
    const ETypes ty(types);
    const u32 T = ty.T, nb = dir == 2 ? 2 : 1;
    EArgs A{d_src, d_tgt, ty.d.ptr, n, n * nb * T * 2, 0, T, nb, dir};
    const u32 grid = (u32)ctx().num_sms * 8;
    DevBuf<u64> out(n + 1);
    if (n == 0) {
        out.zero();
        d2h(out_p, out.ptr, 1);
        sync_stream();
        return 0;
    }
    EeBatch B(A);
    // Compulsory bytes ("edge_expand"): 16 per list (its row pointers), 12 per forward entry (column + value), 28 per reverse
    // entry (column 4, plus its forward point lookup: row pointers 16, value 8), 4 per entry of the delta-minus rows searched,
    // and 14 per output entry (node 4, id 8, type 2), 15 with the direction.
    TimedScope ts(TK_EDGE_EXPAND, 0);
    B.prepare(mode, grid);
    A = B.A;
    LAUNCH(k_ee_rowptr, grid_for(n + 1, 256, grid), 256, 0, A, B.lstart.ptr, B.pos.ptr, out.ptr);
    d2h(out_p, out.ptr, n + 1);
    sync_stream();
    const u64 total = out_p[n];
    ts.bytes = B.bytes() + (out_rev ? 15 : 14) * total;
    if (total > capacity || total == 0) return total;
    DevBuf<u32> dnode(total);
    DevBuf<u64> dedge(total);
    DevBuf<uint16_t> dtype;
    DevBuf<uint8_t> drev;
    if (out_type) dtype.alloc(total);
    if (out_rev) drev.alloc(total);
    LAUNCH(k_ee_fill, grid_for(A.E, 256, grid), 256, 0, A, B.lstart.ptr, B.lo.ptr, B.llen.ptr, B.val.ptr, B.fin, B.pos.ptr, dnode.ptr,
           dedge.ptr, dtype.ptr, drev.ptr);
    d2h(out_node, dnode.ptr, total);
    d2h(out_edge, dedge.ptr, total);
    if (out_type) d2h(out_type, dtype.ptr, total);
    if (out_rev) d2h(out_rev, drev.ptr, total);
    sync_stream();
    return total;
}

} // namespace b200
