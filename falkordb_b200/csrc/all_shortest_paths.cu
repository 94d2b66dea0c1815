// all_shortest_paths.cu -- allShortestPaths((a)-[:R1|R2*..k]->(b)) for a batch of bound pairs (B200_all_shortest_paths): every
// shortest path of each pair, in the order the reference's AllShortestPathsOp::expand_row emits them (all_shortest_paths.rs:82-302).
//
// The sequential statement.  A FIFO BFS from src over get_node_relationships_by_type's adjacency records, for every vertex, the
// entries that reach it from the level before (its predecessors, in visit order); a DFS from dst pushes a node's predecessors in
// list order, so the last one pops first.  The same thing, level-synchronous, per pair (a slot):
// Forward.  Give each front entry its rank (its position in the front).  Level L + 1 is the set of unseen far ends of level L's
// adjacency entries, ordered by the (rank, adjacency position) of the first entry that reaches them.  So a level emits one
// candidate per (front entry, adjacency entry) keyed (slot << 32 | v), sorts it stably (candidates are emitted in (rank,
// position) order, so the first of a run is the first to reach v), keeps the first of each run and re-sorts those by position.
// A slot stops after the first level that has an entry into dst (for src == dst: back into src), at max_hops, or on an empty
// front.  Each level is stored as its (slot << 32 | v) keys, ascending, with their ranks.
// Backward.  The predecessors of v at depth l + 1 are all entries from depth-l nodes to v, in (rank(u), type, half, id) order,
// where half is 0 when the entry is in u's outgoing half.  From dst, level by level, the reverse adjacency of the ancestor set
// (incoming edges for an outgoing pattern; both halves, seen from the far end, for a bidirectional one) is fetched; entries whose
// far end u sits in the stored level l are kept and sorted stably by (rank(u), type, half), then by ancestor.  The distinct u are
// the next ancestor set.  So this costs the ancestors' in-degree, not a second forward sweep.
// Counts and order.  cnt(src) = 1 and cnt(v) = the saturating sum of its predecessors' counts; per predecessor j of v the suffix
// sum suf[j] over j and the predecessors after it.  Path r of a pair (DFS order) is unranked from dst: the predecessor taken is
// the last j with r < suf[j], and r drops by suf[j + 1].  A saturated suffix is only ever taken, never subtracted, so the walk is
// exact for every r below 2^64 - 1.
#include "edge_layers.cuh"

namespace b200 {

// one ancestor level of the backward phase: keys ascending; predecessors of key a at ps[a] .. ps[a+1], each with its ancestor
// index pu in the level below, its relationship id and its suffix count; cnt[a] = suf[ps[a]] (level 0: 1)
struct AsBack { const u64 *key; u64 n; const u64 *ps; const u32 *pu; const u64 *pedge; const u64 *suf; const u64 *cnt; };

__global__ void k_as_seed(const u64 *__restrict__ src, u64 S, u64 nw, u64 *__restrict__ front, u64 *__restrict__ vis) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        const u32 v = (u32)src[s];
        front[s] = s << 32 | v;
        vis[s * nw + (v >> 6)] |= 1ULL << (v & 63);
    }
}
// candidate q of the piece (global position g = q0 + q, in (rank, adjacency position) order): kept with key (slot << 32 | v) when
// the slot has not seen v, else SLOT_NONE; an entry into the slot's dst marks the slot found
__global__ void k_as_emit(const u64 *__restrict__ front, const u64 *__restrict__ cum, u64 i0, u64 i1, u64 q0, u64 R,
                          const u32 *__restrict__ row, const u64 *__restrict__ adj_p, const u32 *__restrict__ adj_node,
                          const u64 *__restrict__ dst, const u64 *__restrict__ vis, u64 nw, u32 *__restrict__ found,
                          u64 *__restrict__ key, u64 *__restrict__ val, u64 *__restrict__ nkept) {
    u64 kept = 0;
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < R; q += (u64)gridDim.x * blockDim.x) {
        const u64 g = q0 + q;
        const u64 a = i0 + list_at(cum + i0, i1 - i0, g);     // the last front entry with cum <= g
        const u64 s = front[a] >> 32;
        const u32 v = adj_node[adj_p[row[a]] + (g - cum[a])];
        if (v == (u32)dst[s]) found[s] = 1;
        const bool live = !slot_seen(vis, nw, s, v);
        key[q] = live ? (s << 32 | v) : SLOT_NONE;
        val[q] = g;
        kept += live;
    }
    if (kept) atomicAdd((unsigned long long *)nkept, (unsigned long long)kept);
}

// the first candidate of each (slot, v) run: marked seen, and (position, key) for the re-sort by position
__global__ void k_as_first(const u64 *__restrict__ key, const u64 *__restrict__ val, u64 E, const u32 *__restrict__ head,
                           const u64 *__restrict__ hpos, u64 *__restrict__ vis, u64 nw, u64 *__restrict__ rk, u64 *__restrict__ nk) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x) {
        if (!head[e]) continue;
        const u64 k = key[e], s = k >> 32;
        const u32 v = (u32)k;
        atomicOr((unsigned long long *)&vis[s * nw + (v >> 6)], 1ULL << (v & 63));
        rk[hpos[e]] = val[e];
        nk[hpos[e]] = k;
    }
}

// the end of a level: a slot found this level stops at depth L + 1
__global__ void k_as_stop(u64 S, const u32 *__restrict__ found, u32 L1, u32 *__restrict__ sdep) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x)
        if (found[s] && !sdep[s]) sdep[s] = L1;
}
// next-front entries of slots still searching (flag[n] = 0)
__global__ void k_as_live(const u64 *__restrict__ front, u64 n, const u32 *__restrict__ sdep, u32 *__restrict__ flag) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (u64)gridDim.x * blockDim.x)
        flag[i] = i < n && !sdep[front[i] >> 32] ? 1 : 0;
}

// backward candidate q (ancestor a, its reverse-adjacency entry): kept when the far end u is in forward level l - 1 of the slot,
// with sort key (rank(u), type, half as u sees it).  A reverse entry of v's outgoing half is in u's incoming half, except a
// self-loop (u == v), which is listed once, in the outgoing half.
__global__ void k_as_back(const u64 *__restrict__ akey, const u64 *__restrict__ cum, u64 na, u64 C, const u32 *__restrict__ row,
                          const u64 *__restrict__ adj_p, const u32 *__restrict__ adj_node, const u32 *__restrict__ adj_tb,
                          const u64 *__restrict__ fkey, const u64 *__restrict__ frank, u64 fn, u32 *__restrict__ keep,
                          u64 *__restrict__ k1) {
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < C; q += (u64)gridDim.x * blockDim.x) {
        const u64 a = list_at(cum, na, q), k = akey[a], s = k >> 32;
        const u64 pos = adj_p[row[a]] + (q - cum[a]);
        const u32 x = adj_node[pos], tb = adj_tb[pos];
        const u64 uk = s << 32 | x, f = lb64(fkey, 0, fn, uk);
        const bool in = f < fn && fkey[f] == uk;
        keep[q] = in;
        if (in) k1[q] = frank[f] << 18 | (u64)(tb >> 1) << 1 | (!(tb & 1) && x != (u32)k ? 1 : 0);
    }
}
__global__ void k_as_pack(const u32 *__restrict__ keep, const u64 *__restrict__ kpos, const u64 *__restrict__ k1, u64 C,
                          u64 *__restrict__ ok1, u64 *__restrict__ oq) {
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < C; q += (u64)gridDim.x * blockDim.x)
        if (keep[q]) { ok1[kpos[q]] = k1[q]; oq[kpos[q]] = q; }
}
__global__ void k_as_anc(const u64 *__restrict__ q, u64 E, const u64 *__restrict__ cum, u64 na, u64 *__restrict__ a) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < E; j += (u64)gridDim.x * blockDim.x) a[j] = list_at(cum, na, q[j]);
}
// predecessor j (final order): its relationship id and far end key; ps[a] = the first predecessor of ancestor a (a = na: E)
__global__ void k_as_preds(const u64 *__restrict__ q, const u64 *__restrict__ anc, u64 E, const u64 *__restrict__ akey,
                           const u64 *__restrict__ cum, const u32 *__restrict__ row, const u64 *__restrict__ adj_p,
                           const u32 *__restrict__ adj_node, const u64 *__restrict__ adj_edge, u64 *__restrict__ pedge,
                           u64 *__restrict__ pkey) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < E; j += (u64)gridDim.x * blockDim.x) {
        const u64 a = anc[j], pos = adj_p[row[a]] + (q[j] - cum[a]);
        pedge[j] = adj_edge[pos];
        pkey[j] = (akey[a] >> 32) << 32 | adj_node[pos];
    }
}
__global__ void k_as_ps(const u64 *__restrict__ anc, u64 E, u64 na, u64 *__restrict__ ps) {
    for (u64 a = (u64)blockIdx.x * blockDim.x + threadIdx.x; a <= na; a += (u64)gridDim.x * blockDim.x) ps[a] = lb64(anc, 0, E, a);
}
// pu[j] = the position of predecessor j's far end in the ancestor level below
__global__ void k_as_pu(const u64 *__restrict__ pkey, u64 E, const u64 *__restrict__ key, u64 n, u32 *__restrict__ pu) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < E; j += (u64)gridDim.x * blockDim.x) pu[j] = (u32)lb64(key, 0, n, pkey[j]);
}

// counts, top-down: per ancestor of level l >= 1 the saturating suffix sums of its predecessors' counts
__global__ void k_as_count(u64 n, const u64 *__restrict__ ps, const u32 *__restrict__ pu, const u64 *__restrict__ below,
                           u64 *__restrict__ suf, u64 *__restrict__ cnt) {
    for (u64 a = (u64)blockIdx.x * blockDim.x + threadIdx.x; a < n; a += (u64)gridDim.x * blockDim.x) {
        u64 c = 0;
        for (u64 j = ps[a + 1]; j-- > ps[a];) {
            const u64 x = below[pu[j]];
            c = c + x < c ? SLOT_NONE : c + x;
            suf[j] = c;
        }
        cnt[a] = c;
    }
}
__global__ void k_as_total(u64 S, const u32 *__restrict__ sdep, const u64 *__restrict__ dst, const AsBack *__restrict__ B,
                           u64 *__restrict__ count, u64 *__restrict__ dpos) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        u64 c = 0, p = 0;
        if (sdep[s]) {
            const AsBack &L = B[sdep[s]];
            p = lb64(L.key, 0, L.n, s << 32 | (u32)dst[s]);
            c = L.cnt[p];
        }
        count[s] = c; dpos[s] = p;
    }
}

// one thread per written path w: pair i (woff[i] <= w < woff[i+1]), rank r = first[i] + w - woff[i], unranked from dst.  Edges
// at eoff[i] + (w - woff[i]) * len, nodes at that + w (len + 1 per path).  src -> dst walk order; for src == dst the list starts
// with the closing edge, as the reference keeps the predecessor chain's order for cycles.
__global__ void k_as_fill(u64 W, u64 S, const u64 *__restrict__ woff, const u64 *__restrict__ first, const u64 *__restrict__ eoff,
                          const u32 *__restrict__ sdep, const u64 *__restrict__ src, const u64 *__restrict__ dst,
                          const u64 *__restrict__ dpos, const AsBack *__restrict__ B, u64 *__restrict__ path_edge,
                          u32 *__restrict__ path_node) {
    for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < W; w += (u64)gridDim.x * blockDim.x) {
        u64 a = 0, b = S - 1;                               // the last pair with woff <= w
        while (a < b) { u64 mid = (a + b + 1) >> 1; if (woff[mid] <= w) a = mid; else b = mid - 1; }
        const u64 s = a, k = w - woff[s], L = sdep[s];
        u64 r = first[s] + k;
        u64 *E = path_edge + eoff[s] + k * L;
        u32 *N = path_node + eoff[s] + k * L + w;
        const bool cyc = src[s] == dst[s];
        u64 x = dpos[s];
        for (u64 l = L; l >= 1; l--) {
            const AsBack &P = B[l];
            const u64 lo = P.ps[x], hi = P.ps[x + 1];
            u64 c = lo, d = hi;                             // the first j with suf[j] <= r (suf is non-increasing)
            while (c < d) { u64 mid = (c + d) >> 1; if (P.suf[mid] <= r) d = mid; else c = mid + 1; }
            const u64 j = c - 1;
            if (j + 1 < hi) r -= P.suf[j + 1];
            x = P.pu[j];
            const u32 u = (u32)B[l - 1].key[x];
            if (cyc) { E[L - l] = P.pedge[j]; N[L - l + 1] = u; }
            else { E[l - 1] = P.pedge[j]; N[l - 1] = u; }
        }
        N[cyc ? 0 : L] = (u32)dst[s];
    }
}

// ---- host side ----

struct AsLevel { DevBuf<u64> key, rank; u64 n = 0; };       // a forward level: its keys ascending, each with its rank
struct AsAnc {                                              // a backward ancestor level (AsBack's arrays)
    DevBuf<u64> key, ps, pedge, pkey, suf, cnt;
    DevBuf<u32> pu;
    u64 n = 0, np = 0;
};

u64 all_shortest_paths(const u64 *h_src, const u64 *h_dst, u64 np, const std::vector<EdgeTypeDev> &types, int dir, u64 n,
                       u64 max_hops, u64 budget, const u64 *h_first, u64 *count, u32 *len, u64 *out_p, u64 *path_edge,
                       u32 *path_node, u64 edge_capacity, u64 *nedges) {
    const ETypes ty(types);
    const int rdir = dir == 0 ? 1 : 2;                      // the reverse adjacency: incoming edges, or both halves
    const u64 nw = (n + 63) / 64;
    size_t fr = 0, tot = 0;
    CUDA_TRY(cudaMemGetInfo(&fr, &tot));
    budget = piece_budget(budget, fr);
    const u64 S_max = std::max<u64>(1, std::min<u64>(1024, fr / 4 / (nw * 8)));
    // Compulsory bytes ("all_shortest_paths"): the adjacency fetches (edge_expand's formula plus 12 per entry written, 16 with the
    // type and half) and 24 per fetched key (its node, row and length); per forward candidate 28 (its neighbour, the visited word,
    // key and position) and per new vertex 40 (the visited word, its position and key, the stored key and rank); per backward
    // candidate 24 (neighbour, type and half, the forward level's rank) and per predecessor 64 (sort keys and position, id, far
    // end key, ancestor index, suffix count and the count it reads); per written path 16 per edge (id and a suffix count) and 4
    // per node.
    TimedScope ts(TK_ALL_SHORTEST_PATHS, 0);
    u64 bytes = 0, flops = 0;
    const u64 cap = path_edge ? edge_capacity : 0;
    u64 e_used = 0, w_used = 0;                             // edges and paths written so far
    bool full = !path_edge;                                 // filling stopped (or count only)
    auto run_slice = [&](u64 p0, u64 S) {
        DevBuf<u64> dsrc(S), ddst(S);
        h2d(dsrc.ptr, h_src + p0, S);
        h2d(ddst.ptr, h_dst + p0, S);
        DevBuf<u64> vis(S * nw), front(S);
        vis.zero();
        LAUNCH(k_as_seed, grid_for(S, PAIR_T), PAIR_T, 0, dsrc.ptr, S, nw, front.ptr, vis.ptr);
        DevBuf<u32> found(S), sdep(S);
        found.zero(); sdep.zero();
        std::vector<AsLevel> lev;
        u64 nf = S;
        // ---- forward levels
        for (u64 L = 0; L < max_hops && nf; L++) {
            if (nf >= ((u64)1 << 32)) throw GrbError(-8, "all_shortest_paths: a level of 2^32 entries");   // ranks are 32 bits
            lev.emplace_back();
            AsLevel &F = lev.back();
            F.n = nf;
            F.key.alloc(nf); F.rank.alloc(nf);
            d2d(F.key.ptr, front.ptr, nf);
            iota_u64(F.rank.ptr, nf);
            sort_pairs_u64(F.key.ptr, F.rank.ptr, nf, SLOT_KEY_BITS);
            bytes += 16 * nf;
            NodeAdj A;
            A.fetch(ty, front.ptr, nf, dir, false, &bytes);
            const u64 total = A.total;
            flops += total;
            bytes += 24 * nf;
            DevBuf<u64> next(1), scal(1);
            u64 nnext = 0;
            for_each_piece(A.cum.ptr, nf, total, budget, [&](u64 i0, u64 i1, u64 q0, u64 q1) {
                const u64 R = q1 - q0;
                DevBuf<u64> key(R), val(R);
                CUDA_TRY(cudaMemsetAsync(scal.ptr, 0, sizeof(u64), stream()));
                LAUNCH(k_as_emit, grid_for(R, PAIR_T, 8 * (u64)ctx().num_sms), PAIR_T, 0, front.ptr, A.cum.ptr, i0, i1, q0, R, A.row.ptr,
                       A.p.ptr, A.node.ptr, ddst.ptr, vis.ptr, nw, found.ptr, key.ptr, val.ptr, scal.ptr);
                const u64 E = read_scalar(scal.ptr);
                bytes += 28 * R;
                if (!E) return;
                sort_pairs_u64(key.ptr, val.ptr, R, SLOT_KEY_BITS);            // stable: the first to reach v leads its run
                DevBuf<u32> head(E + 1);
                DevBuf<u64> hpos(E + 1);
                const u64 nh = run_heads(key.ptr, E, head.ptr, hpos.ptr);
                DevBuf<u64> rk(nh), nk(nh);
                LAUNCH(k_as_first, grid_for(E, PAIR_T), PAIR_T, 0, key.ptr, val.ptr, E, head.ptr, hpos.ptr, vis.ptr, nw, rk.ptr, nk.ptr);
                sort_pairs_u64(rk.ptr, nk.ptr, nh, bit_length(total));         // by (rank, adjacency position)
                grow(next, nnext, nnext + nh);
                d2d(next.ptr + nnext, nk.ptr, nh);
                nnext += nh;
                bytes += 40 * nh;
            });
            LAUNCH(k_as_stop, grid_for(S, PAIR_T), PAIR_T, 0, S, found.ptr, (u32)(L + 1), sdep.ptr);
            DevBuf<u32> flag(nnext + 1);
            DevBuf<u64> fpos(nnext + 1);
            LAUNCH(k_as_live, grid_for(nnext + 1, PAIR_T), PAIR_T, 0, next.ptr, nnext, sdep.ptr, flag.ptr);
            exclusive_scan_u32_to_u64(flag.ptr, fpos.ptr, nnext + 1);
            nf = read_scalar(fpos.ptr + nnext);
            front.alloc(std::max<u64>(nf, 1));
            if (nf) scatter_flagged(next.ptr, nnext, flag.ptr, fpos.ptr, front.ptr);
        }
        front.release(); vis.release();
        std::vector<u32> hdep(S);
        d2h(hdep.data(), sdep.ptr, S);
        sync_stream();
        u64 Lmax = 0;
        for (u32 d : hdep) Lmax = std::max<u64>(Lmax, d);
        // ---- backward levels, from the deepest dst down to the srcs
        std::vector<AsAnc> anc(Lmax + 1);
        DevBuf<u64> carry;                                  // the far ends of the level above's predecessors
        u64 ncarry = 0;
        for (u64 l = Lmax + 1; l-- > 0;) {
            AsAnc &Y = anc[l];
            std::vector<u64> seeds;
            for (u64 s = 0; s < S; s++) if (hdep[s] == l && l) seeds.push_back(s << 32 | h_dst[p0 + s]);
            Y.key.alloc(ncarry + seeds.size());
            d2d(Y.key.ptr, carry.ptr, ncarry);
            h2d(Y.key.ptr + ncarry, seeds.data(), seeds.size());
            Y.n = unique_sorted(Y.key, ncarry + seeds.size(), SLOT_KEY_BITS);
            carry.release(); ncarry = 0;
            if (l + 1 <= Lmax && anc[l + 1].np)             // the level above's predecessors, as positions in this level
                LAUNCH(k_as_pu, grid_for(anc[l + 1].np, PAIR_T), PAIR_T, 0, anc[l + 1].pkey.ptr, anc[l + 1].np, Y.key.ptr, Y.n,
                       anc[l + 1].pu.ptr);
            if (l + 1 <= Lmax) anc[l + 1].pkey.release();
            if (l == 0 || !Y.n) continue;
            NodeAdj A;
            A.fetch(ty, Y.key.ptr, Y.n, rdir, true, &bytes);
            const u64 C = A.total;
            bytes += 24 * Y.n;
            flops += C;
            DevBuf<u32> keep(C + 1);
            DevBuf<u64> k1(std::max<u64>(C, 1)), kpos(C + 1);
            CUDA_TRY(cudaMemsetAsync(keep.ptr + C, 0, sizeof(u32), stream()));
            const AsLevel &F = lev[l - 1];
            if (C) LAUNCH(k_as_back, grid_for(C, PAIR_T), PAIR_T, 0, Y.key.ptr, A.cum.ptr, Y.n, C, A.row.ptr, A.p.ptr, A.node.ptr, A.tb.ptr,
                          F.key.ptr, F.rank.ptr, F.n, keep.ptr, k1.ptr);
            exclusive_scan_u32_to_u64(keep.ptr, kpos.ptr, C + 1);
            const u64 E = read_scalar(kpos.ptr + C);
            bytes += 24 * C + 64 * E;
            Y.np = E;
            Y.ps.alloc(Y.n + 1); Y.pedge.alloc(E); Y.pkey.alloc(E); Y.pu.alloc(E); Y.suf.alloc(E);
            DevBuf<u64> sk(E), sq(E);
            if (E) {
                LAUNCH(k_as_pack, grid_for(C, PAIR_T), PAIR_T, 0, keep.ptr, kpos.ptr, k1.ptr, C, sk.ptr, sq.ptr);
                keep.release(); k1.release(); kpos.release();
                sort_pairs_u64(sk.ptr, sq.ptr, E, bit_length(F.n) + 18);           // (rank(u), type, half), stable on position
                LAUNCH(k_as_anc, grid_for(E, PAIR_T), PAIR_T, 0, sq.ptr, E, A.cum.ptr, Y.n, sk.ptr);
                sort_pairs_u64(sk.ptr, sq.ptr, E, bit_length(Y.n));               // then by ancestor, stable
                LAUNCH(k_as_preds, grid_for(E, PAIR_T), PAIR_T, 0, sq.ptr, sk.ptr, E, Y.key.ptr, A.cum.ptr, A.row.ptr, A.p.ptr, A.node.ptr,
                       A.edge.ptr, Y.pedge.ptr, Y.pkey.ptr);
            }
            LAUNCH(k_as_ps, grid_for(Y.n + 1, PAIR_T), PAIR_T, 0, sk.ptr, E, Y.n, Y.ps.ptr);
            carry.alloc(E);
            d2d(carry.ptr, Y.pkey.ptr, E);
            ncarry = E;
        }
        // ---- counts, top-down, and each pair's total
        std::vector<AsBack> hb(Lmax + 1);
        for (u64 l = 0; l <= Lmax; l++) {
            AsAnc &Y = anc[l];
            Y.cnt.alloc(std::max<u64>(Y.n, 1));
            if (l == 0) { if (Y.n) fill_u64(Y.cnt.ptr, 1, Y.n); }
            else if (Y.n) LAUNCH(k_as_count, grid_for(Y.n, PAIR_T), PAIR_T, 0, Y.n, Y.ps.ptr, Y.pu.ptr, anc[l - 1].cnt.ptr, Y.suf.ptr, Y.cnt.ptr);
            hb[l] = AsBack{Y.key.ptr, Y.n, Y.ps.ptr, Y.pu.ptr, Y.pedge.ptr, Y.suf.ptr, Y.cnt.ptr};
        }
        DevBuf<AsBack> db(Lmax + 1);
        h2d(db.ptr, hb.data(), Lmax + 1);
        DevBuf<u64> dcount(S), dpos(S);
        LAUNCH(k_as_total, grid_for(S, PAIR_T), PAIR_T, 0, S, sdep.ptr, ddst.ptr, db.ptr, dcount.ptr, dpos.ptr);
        std::vector<u64> hcount(S);
        d2h(hcount.data(), dcount.ptr, S);
        sync_stream();
        // ---- the window of each pair: from first[i] on, while whole paths fit
        std::vector<u64> woff(S + 1, 0), eoff(S, 0), hfirst(S, 0);
        u64 e = e_used;
        bool stop = full;
        for (u64 s = 0; s < S; s++) {
            const u64 f = h_first ? h_first[p0 + s] : 0, avail = hcount[s] > f ? hcount[s] - f : 0, L = hdep[s];
            u64 w = 0;
            if (!stop && avail) {
                w = std::min<u64>(avail, (cap - e) / L);
                if (w < avail) stop = true;
            }
            hfirst[s] = f; eoff[s] = e - e_used; woff[s + 1] = woff[s] + w;
            e += w * L;
        }
        const u64 W = woff[S], ne = e - e_used;
        if (W) {
            DevBuf<u64> dwoff(S + 1), dfirst(S), deoff(S), oedge(ne);
            DevBuf<u32> onode(ne + W);
            h2d(dwoff.ptr, woff.data(), S + 1); h2d(dfirst.ptr, hfirst.data(), S); h2d(deoff.ptr, eoff.data(), S);
            LAUNCH(k_as_fill, grid_for(W, PAIR_T), PAIR_T, 0, W, S, dwoff.ptr, dfirst.ptr, deoff.ptr, sdep.ptr, dsrc.ptr, ddst.ptr, dpos.ptr,
                   db.ptr, oedge.ptr, onode.ptr);
            d2h(path_edge + e_used, oedge.ptr, ne);
            d2h(path_node + e_used + w_used, onode.ptr, ne + W);
            sync_stream();
            bytes += 16 * ne + 4 * (ne + W);
        }
        // committed only now: a slice rerun after running out of memory starts from the same state
        for (u64 s = 0; s < S; s++) {
            count[p0 + s] = hcount[s];
            len[p0 + s] = hdep[s];
            out_p[p0 + s] = w_used + woff[s];
        }
        e_used += ne; w_used += W; full = stop;
    };
    for_each_slice(np, S_max, run_slice);
    out_p[np] = w_used;
    *nedges = e_used;
    ts.bytes = bytes;
    return flops;
}

} // namespace b200
