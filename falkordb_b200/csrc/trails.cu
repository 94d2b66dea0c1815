// trails.cu -- CondVarLenTraverse's trails (cond_var_len_traverse.rs:152-386) for a batch of start nodes in one call
// (B200_var_len_trails): every relationship-unique path of min_hops..max_hops edges, in the reference's emission order.
//
// Levels.  Level 0 holds the starts; level h >= 1 holds the trail-tree entries (parent, node, edge) of h edges.  Since
// will_continue is hop < max_hops whatever else holds (:319), every trail of fewer than max_hops edges continues and is stored; the
// last level (hop == max_hops) only emits, is counted per parent and written straight to the output.  Entries are stored in parent
// order, so the children of an entry are contiguous: cb[e] .. cb[e+1] of the next level.
// Expansion of level h.  The adjacency of the level's distinct nodes is fetched once (edge_adjacency: edges.cu's lists, counts and
// scan, placed in get_node_relationships_by_type's order).  One thread per (entry, adjacency position), found from the scan of the
// entries' adjacency lengths, drops an edge already on the trail (a walk up the parent chain, h reads), sets will_emit as :314-317
// (hop >= min_hops, the fixed destination, the destination-label bitmap) and is kept (stored, or emitted on the last level).
// Order.  Per start: the 0-hop emission, then block(root); block(X) = X's emitting children in adjacency order, then block(c) for
// each continuing child c in reverse adjacency order (frames are pushed in adjacency order and popped last-first, :380-383).  With
// S(X) = |block(X)| computed bottom-up (segmented sums over the contiguous children), positions follow top-down: the emitting child
// of rank k sits at P(X) + k, the continuing child c at P(X) + ecount(X) + the sizes of the blocks of X's children after c.
#include "edge_layers.cuh"

namespace b200 {

struct TLev { const u64 *par; const u32 *node; const u64 *edge; };   // level 0: node only (the starts)
struct TArgs {
    const TLev *lev;           // levels 0 .. h
    const i64 *dests;          // per start, < 0: none; null: none
    const u32 *lab;            // destination-label bitmap; null: every node
    u64 min_hops, max_hops;
};

__device__ __forceinline__ bool can_end(const TArgs &T, u64 root, u32 x) {
    if (T.dests && T.dests[root] >= 0 && (u64)T.dests[root] != x) return false;
    return !T.lab || ((T.lab[x >> 5] >> (x & 31)) & 1);
}
// the node and edge id of candidate q of level h (entry e at adjacency position q - cstart[e])
__device__ __forceinline__ u64 cand_at(const u64 *__restrict__ cstart, u64 n, const u32 *__restrict__ slot,
                                       const u64 *__restrict__ adj_p, u64 q, u64 *e) {
    *e = list_at(cstart, n, q);
    return adj_p[slot[*e]] + (q - cstart[*e]);
}
// the trail ending at entry c of level lv, written in walk order from the start: edges at eb .. eb + lv, nodes at nb .. nb + lv
__device__ __forceinline__ void write_path(const TArgs &T, u32 lv, u64 c, u64 eb, u64 nb, u64 *__restrict__ path_edge,
                                           u32 *__restrict__ path_node) {
    for (u32 l = lv; l >= 1; l--) {
        path_edge[eb + l - 1] = T.lev[l].edge[c];
        path_node[nb + l] = T.lev[l].node[c];
        c = T.lev[l].par[c];
    }
    path_node[nb] = T.lev[0].node[c];
}

// AND of the labels' diagonals (m \ dm) u dp into the bitmap (all ones on entry)
__global__ void k_tr_label(ECsr m, ECsr dp, ECsr dm, u64 n, u32 *__restrict__ bits) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (u64)gridDim.x * blockDim.x) {
        const bool has = find_rc(dp, r, (u32)r) != ~0ULL || (find_rc(m, r, (u32)r) != ~0ULL && find_rc(dm, r, (u32)r) == ~0ULL);
        if (!has) atomicAnd(&bits[r >> 5], ~(1u << (r & 31)));
    }
}

// per start: the 0-hop emission (:159-170)
__global__ void k_tr_zero(TArgs T, u64 n, u32 *__restrict__ z) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        z[i] = T.min_hops == 0 && can_end(T, i, T.lev[0].node[i]) ? 1 : 0;
}

// per candidate of level h (hop = h + 1): kept (stored, or on the last level emitted) and will_emit
__global__ void k_tr_cand(TArgs T, u32 h, const u64 *__restrict__ cstart, u64 n, const u32 *__restrict__ slot,
                          const u64 *__restrict__ adj_p, const u32 *__restrict__ adj_node, const u64 *__restrict__ adj_edge, u64 C,
                          u32 *__restrict__ kept, u32 *__restrict__ emit) {
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < C; q += (u64)gridDim.x * blockDim.x) {
        u64 e;
        const u64 a = cand_at(cstart, n, slot, adj_p, q, &e);
        const u64 id = adj_edge[a];
        u64 cur = e;
        bool used = false;
        for (u32 l = h; l >= 1; l--) {                                        // relationship uniqueness (:248-251)
            if (T.lev[l].edge[cur] == id) { used = true; break; }
            cur = T.lev[l].par[cur];
        }
        u32 k = 0, em = 0;
        if (!used) {
            const u64 hop = (u64)h + 1;
            em = hop >= T.min_hops && can_end(T, cur, adj_node[a]) ? 1 : 0;
            k = hop < T.max_hops ? 1 : em;
        }
        kept[q] = k;
        if (emit) emit[q] = em;
    }
}

// cb[e] = the first kept candidate of entry e (e = n: the total)
__global__ void k_tr_cb(const u64 *__restrict__ cstart, const u64 *__restrict__ kpos, u64 n, u64 *__restrict__ cb) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e <= n; e += (u64)gridDim.x * blockDim.x) cb[e] = kpos[cstart[e]];
}

// the kept candidates of level h become level h + 1
__global__ void k_tr_fill(const u64 *__restrict__ cstart, u64 n, const u32 *__restrict__ slot, const u64 *__restrict__ adj_p,
                          const u32 *__restrict__ adj_node, const u64 *__restrict__ adj_edge, u64 C, const u32 *__restrict__ kept,
                          const u32 *__restrict__ emit, const u64 *__restrict__ kpos, u64 *__restrict__ par, u32 *__restrict__ node,
                          u64 *__restrict__ edge, u32 *__restrict__ cemit) {
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < C; q += (u64)gridDim.x * blockDim.x) {
        if (!kept[q]) continue;
        u64 e;
        const u64 a = cand_at(cstart, n, slot, adj_p, q, &e), c = kpos[q];
        par[c] = e; node[c] = adj_node[a]; edge[c] = adj_edge[a]; cemit[c] = emit[q];
    }
}

// bottom-up: S(e) = ecount(e) + the S of its stored children (+ the 0-hop emission at level 0).  cb null: no children;
// cemp null: the children are last-level emissions (every kept one emits), else cemp / cprefS = the child level's scans.
__global__ void k_tr_sum(u64 n, const u64 *__restrict__ cb, const u64 *__restrict__ cemp, const u64 *__restrict__ cprefS,
                         const u32 *__restrict__ z, u64 *__restrict__ S) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (u64)gridDim.x * blockDim.x) {
        u64 s = z ? z[e] : 0;
        if (cb) {
            const u64 a = cb[e], b = cb[e + 1];
            s += cemp ? cemp[b] - cemp[a] + cprefS[b] - cprefS[a] : b - a;
        }
        S[e] = s;
    }
}

// top-down: P(c) for the entries c of level h + 1 from their parents' P (level h)
__global__ void k_tr_pos(u64 n, const u64 *__restrict__ par, const u64 *__restrict__ pcb, const u64 *__restrict__ pP,
                         const u64 *__restrict__ emp, const u64 *__restrict__ prefS, u64 *__restrict__ P) {
    for (u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (u64)gridDim.x * blockDim.x) {
        const u64 X = par[c], a = pcb[X], b = pcb[X + 1];
        P[c] = pP[X] + (emp[b] - emp[a]) + (prefS[b] - prefS[c + 1]);
    }
}
__global__ void k_tr_pos0(u64 n, const u64 *__restrict__ prefS, const u32 *__restrict__ z, u64 *__restrict__ P) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) P[i] = prefS[i] + z[i];
}

// Emissions.  E null: the end node and hop count of every trail; else (E = the scan of the hop counts) its path.
__global__ void k_tr_out0(TArgs T, u64 n, const u32 *__restrict__ z, const u64 *__restrict__ out_p, u32 *__restrict__ end,
                          u32 *__restrict__ hops, const u64 *__restrict__ E, u32 *__restrict__ path_node) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        if (!z[i]) continue;
        const u64 k = out_p[i];
        if (!E) { end[k] = T.lev[0].node[i]; hops[k] = 0; }
        else path_node[E[k] + k] = T.lev[0].node[i];
    }
}
__global__ void k_tr_out(TArgs T, u32 lv, u64 n, const u32 *__restrict__ emit, const u64 *__restrict__ emp, const u64 *__restrict__ pcb,
                         const u64 *__restrict__ pP, u32 *__restrict__ end, u32 *__restrict__ hops, const u64 *__restrict__ E,
                         u64 *__restrict__ path_edge, u32 *__restrict__ path_node) {
    for (u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x; c < n; c += (u64)gridDim.x * blockDim.x) {
        if (!emit[c]) continue;
        const u64 X = T.lev[lv].par[c], k = pP[X] + emp[c] - emp[pcb[X]];
        if (!E) { end[k] = T.lev[lv].node[c]; hops[k] = lv; }
        else write_path(T, lv, c, E[k], E[k] + k, path_edge, path_node);
    }
}
__global__ void k_tr_out_last(TArgs T, u32 h, const u64 *__restrict__ cstart, u64 n, const u32 *__restrict__ slot,
                              const u64 *__restrict__ adj_p, const u32 *__restrict__ adj_node, const u64 *__restrict__ adj_edge, u64 C,
                              const u32 *__restrict__ kept, const u64 *__restrict__ kpos, const u64 *__restrict__ cb,
                              const u64 *__restrict__ P, u32 *__restrict__ end, u32 *__restrict__ hops, const u64 *__restrict__ E,
                              u64 *__restrict__ path_edge, u32 *__restrict__ path_node) {
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < C; q += (u64)gridDim.x * blockDim.x) {
        if (!kept[q]) continue;
        u64 e;
        const u64 a = cand_at(cstart, n, slot, adj_p, q, &e), k = P[e] + kpos[q] - cb[e];
        if (!E) { end[k] = adj_node[a]; hops[k] = h + 1; }
        else {
            const u64 eb = E[k], nb = eb + k;
            path_edge[eb + h] = adj_edge[a];
            path_node[nb + h + 1] = adj_node[a];
            write_path(T, h, e, eb, nb, path_edge, path_node);
        }
    }
}

namespace {
struct Level {                  // level h of the trail tree
    u64 n = 0;
    DevBuf<u64> par, edge;      // h >= 1
    DevBuf<u32> node, emit;     // emit: h >= 1
    DevBuf<u64> emp, prefS, P;  // exclusive scans of emit and of S (n + 1); block starts
    DevBuf<u64> cb;             // n + 1: the children of each entry in the next level (or its kept last-level candidates); empty: none
    bool last_children = false; // cb indexes the last level's kept candidates
};
struct LastLevel {              // the expansion of level h into the emit-only hop max_hops (kept for the output passes)
    u32 h = 0; u64 n = 0;
    NodeAdj adj;
    DevBuf<u64> kpos;
    DevBuf<u32> kept;
};
}

int var_len_trails(const u64 *h_starts, const i64 *h_dests, u64 nstarts, const std::vector<EdgeTypeDev> &types, int dir, u64 min_hops,
                   u64 max_hops, const std::vector<LabelDev> &labels, u64 nv, u64 tree_capacity, TrailsOut &o) {
    const u32 grid = (u32)ctx().num_sms * 8;
    const ETypes ty(types);
    std::vector<std::unique_ptr<Level>> lv;
    lv.emplace_back(new Level());
    Level &L0 = *lv[0];
    L0.n = nstarts;
    {
        std::vector<u32> s32(h_starts, h_starts + nstarts);
        L0.node.alloc(nstarts);
        h2d(L0.node.ptr, s32.data(), nstarts);
    }
    DevBuf<i64> ddest;
    if (h_dests) { ddest.alloc(nstarts); h2d(ddest.ptr, h_dests, nstarts); }
    DevBuf<u32> lab;
    // Compulsory bytes ("var_len_trails"): per label, 16 per vertex (the diagonal probes' row pointers) and the bitmap; per level,
    // the adjacency fetch (edge_expand's formula, 12 per adjacency entry written) and 16 per entry (node, slot, candidate start);
    // per candidate 24 (node and id, kept flag and position) + 16 per edge of the parent's trail (the uniqueness walk reads an
    // edge and a parent); 28 per stored entry (parent, node, edge, emit flag); per trail 8 (end and hops), and with paths 12 per
    // path edge and 4 per path node.
    TimedScope ts(TK_VAR_LEN_TRAILS, 0);
    u64 bytes = 0;
    if (!labels.empty()) {
        lab.alloc((nv + 31) / 32);
        CUDA_TRY(cudaMemsetAsync(lab.ptr, 0xff, lab.bytes(), stream()));
        for (const LabelDev &l : labels) {
            LAUNCH(k_tr_label, grid_for(nv, 256, grid), 256, 0, ecsr(l.m), ecsr(l.dp), ecsr(l.dm), nv, lab.ptr);
            bytes += 16 * nv + nv / 8;
        }
    }
    DevBuf<TLev> dlev;
    std::vector<TLev> hlev;
    auto upload_levels = [&]() {
        hlev.clear();
        for (auto &l : lv) hlev.push_back(TLev{l->par.ptr, l->node.ptr, l->edge.ptr});
        dlev.alloc(hlev.size());
        h2d(dlev.ptr, hlev.data(), hlev.size());
    };
    TArgs A{nullptr, ddest.ptr, lab.ptr, min_hops, max_hops};
    upload_levels();
    A.lev = dlev.ptr;
    DevBuf<u32> z(nstarts);
    LAUNCH(k_tr_zero, grid_for(nstarts, 256, grid), 256, 0, A, nstarts, z.ptr);
    LastLevel last;
    bool has_last = false;
    u64 stored = 0, npath = 0;
    // ---- expansion, level by level
    for (u32 h = 0; (u64)h < max_hops && lv[h]->n; h++) {
        Level &X = *lv[h];
        const u64 n = X.n;
        const bool to_last = (u64)h + 1 == max_hops;
        // candidates: one per (entry, adjacency position of its node)
        NodeAdj adj;
        adj.fetch(ty, X.node.ptr, n, dir, false, &bytes);
        const u64 C = adj.total;
        DevBuf<u32> kept(C + 1), emit;
        DevBuf<u64> kpos(C + 1);
        if (!to_last) emit.alloc(C);
        CUDA_TRY(cudaMemsetAsync(kept.ptr + C, 0, sizeof(u32), stream()));
        if (C) LAUNCH(k_tr_cand, grid_for(C, 256, grid), 256, 0, A, h, adj.cum.ptr, n, adj.row.ptr, adj.p.ptr, adj.node.ptr,
                      adj.edge.ptr, C, kept.ptr, emit.ptr);
        exclusive_scan_u32_to_u64(kept.ptr, kpos.ptr, C + 1);
        X.cb.alloc(n + 1);
        LAUNCH(k_tr_cb, grid_for(n + 1, 256, grid), 256, 0, adj.cum.ptr, kpos.ptr, n, X.cb.ptr);
        const u64 K = read_scalar(kpos.ptr + C);
        bytes += 16 * n + C * (24 + 16 * (u64)h);
        if (to_last) {
            X.last_children = true;
            npath += K * max_hops;
            if (o.out_end) {                        // the output passes re-read this level's candidates
                last.h = h; last.n = n;
                last.adj = std::move(adj); last.kpos = std::move(kpos); last.kept = std::move(kept);
                has_last = true;
            }
            break;
        }
        if (stored + K > tree_capacity) return 2;
        stored += K;
        lv.emplace_back(new Level());
        Level &Y = *lv[h + 1];
        Y.n = K;
        Y.par.alloc(K); Y.node.alloc(K); Y.edge.alloc(K); Y.emit.alloc(K + 1); Y.emp.alloc(K + 1);
        CUDA_TRY(cudaMemsetAsync(Y.emit.ptr + K, 0, sizeof(u32), stream()));
        if (K) LAUNCH(k_tr_fill, grid_for(C, 256, grid), 256, 0, adj.cum.ptr, n, adj.row.ptr, adj.p.ptr, adj.node.ptr, adj.edge.ptr,
                      C, kept.ptr, emit.ptr, kpos.ptr, Y.par.ptr, Y.node.ptr, Y.edge.ptr, Y.emit.ptr);
        exclusive_scan_u32_to_u64(Y.emit.ptr, Y.emp.ptr, K + 1);
        npath += read_scalar(Y.emp.ptr + K) * (h + 1);
        bytes += 28 * K;
        upload_levels();
        A.lev = dlev.ptr;
    }
    // ---- block sizes, bottom-up; the roots' sums are out_p
    for (size_t h = lv.size(); h-- > 0;) {
        Level &X = *lv[h];
        Level *Y = h + 1 < lv.size() ? lv[h + 1].get() : nullptr;
        X.prefS.alloc(X.n + 1);
        DevBuf<u64> S(X.n + 1);
        CUDA_TRY(cudaMemsetAsync(S.ptr + X.n, 0, sizeof(u64), stream()));
        const u64 *cb = X.cb.ptr;            // null: level h was not expanded
        if (X.n)
            LAUNCH(k_tr_sum, grid_for(X.n, 256, grid), 256, 0, X.n, cb, X.last_children || !Y ? nullptr : Y->emp.ptr,
                   X.last_children || !Y ? nullptr : Y->prefS.ptr, h == 0 ? z.ptr : nullptr, S.ptr);
        exclusive_scan_u64(S.ptr, X.prefS.ptr, X.n + 1);
    }
    d2h(o.out_p, L0.prefS.ptr, nstarts + 1);
    sync_stream();
    o.nout = o.out_p[nstarts];
    o.npath = npath;
    const bool paths = o.path_edge != nullptr;
    if (!o.out_end || o.nout == 0 || o.nout > o.out_capacity || (paths && npath > o.path_capacity)) {
        ts.bytes = bytes;
        return !o.out_end || o.nout == 0 ? 0 : 1;
    }
    // ---- positions, top-down
    L0.P.alloc(nstarts);
    LAUNCH(k_tr_pos0, grid_for(nstarts, 256, grid), 256, 0, nstarts, L0.prefS.ptr, z.ptr, L0.P.ptr);
    for (size_t h = 1; h < lv.size(); h++) {
        Level &Y = *lv[h], &X = *lv[h - 1];
        Y.P.alloc(Y.n);
        if (Y.n) LAUNCH(k_tr_pos, grid_for(Y.n, 256, grid), 256, 0, Y.n, Y.par.ptr, X.cb.ptr, X.P.ptr, Y.emp.ptr, Y.prefS.ptr, Y.P.ptr);
    }
    // ---- the output: end nodes and hop counts, then (with paths) the walks
    const u64 N = o.nout;
    DevBuf<u32> dend(N), dhops(N + 1), dpnode;
    DevBuf<u64> E, dpedge;
    if (paths) {
        E.alloc(N + 1); dpedge.alloc(npath); dpnode.alloc(npath + N);
        CUDA_TRY(cudaMemsetAsync(dhops.ptr + N, 0, sizeof(u32), stream()));
    }
    for (int pass = 0; pass < (paths ? 2 : 1); pass++) {
        const u64 *e = pass ? E.ptr : nullptr;
        if (pass) exclusive_scan_u32_to_u64(dhops.ptr, E.ptr, N + 1);
        LAUNCH(k_tr_out0, grid_for(nstarts, 256, grid), 256, 0, A, nstarts, z.ptr, L0.prefS.ptr, dend.ptr, dhops.ptr, e, dpnode.ptr);
        for (size_t h = 1; h < lv.size(); h++) {
            Level &Y = *lv[h];
            if (Y.n)
                LAUNCH(k_tr_out, grid_for(Y.n, 256, grid), 256, 0, A, (u32)h, Y.n, Y.emit.ptr, Y.emp.ptr, lv[h - 1]->cb.ptr,
                       lv[h - 1]->P.ptr, dend.ptr, dhops.ptr, e, dpedge.ptr, dpnode.ptr);
        }
        const NodeAdj &LA = last.adj;
        if (has_last && LA.total)
            LAUNCH(k_tr_out_last, grid_for(LA.total, 256, grid), 256, 0, A, last.h, LA.cum.ptr, last.n, LA.row.ptr, LA.p.ptr,
                   LA.node.ptr, LA.edge.ptr, LA.total, last.kept.ptr, last.kpos.ptr, lv[last.h]->cb.ptr, lv[last.h]->P.ptr, dend.ptr,
                   dhops.ptr, e, dpedge.ptr, dpnode.ptr);
    }
    d2h(o.out_end, dend.ptr, N);
    if (o.out_hops) d2h(o.out_hops, dhops.ptr, N);
    if (paths) { d2h(o.path_edge, dpedge.ptr, npath); d2h(o.path_node, dpnode.ptr, npath + N); }
    sync_stream();
    bytes += 8 * N + (paths ? 16 * npath + 4 * N : 0);
    ts.bytes = bytes;
    return 0;
}

} // namespace b200
