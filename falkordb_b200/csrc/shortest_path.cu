// shortest_path.cu -- the shortestPath((a)-[:R1|R2*min..max]->(b)) expression for a batch of bound pairs (B200_shortest_path):
// the reference's bidirectional BFS (bfs_shortest_path, eval.rs:1386-1513), path for path, level-synchronous on the device.
//
// The sequential loop.  Each round expands one whole side: the forward side F when |f_front| <= |b_front|, else the backward side
// B.  Its front is walked in order and each node's neighbours ascending; a neighbour the side has not seen is recorded with that
// node as parent, and is then either a meet candidate (the other side has seen it; kept only if its other-side depth od is
// strictly below the best so far) or appended to the next front.  The round completes before the loop looks at the meet.
// The same thing, level-synchronous.  Give the front's nodes their rank r (their position in the front).  A new v is first met from
// its lowest-ranked front neighbour, so that is its parent; the next front is ordered by (parent rank, v); and the first candidate
// with the least od is the lexicographic minimum of (od, r, v).  So one round is: emit (slot, v, r) for every effective neighbour v
// of every front node not yet seen by the side, a stable sort by (slot, v) (the entries are emitted rank-major, so the first of
// each run holds the least r), the other side's membership of each distinct (slot, v), the segmented minimum of (od, r, v), and the
// survivors re-sorted by r (stable, so v stays ascending inside one r) as the next front.
// Pieces.  When a round's neighbour entries exceed the candidate budget (option "shortest_path_budget"), the front is cut into
// rank-ordered pieces and each piece marks its vertices seen before the next is emitted: a vertex an earlier piece found is not
// found again, exactly as in the sequential walk.  A later piece's meet replaces an earlier one only with a strictly smaller od.
// State.  Pairs run in slices of at most 1024 slots.  Per side: a slot-major visited bitmap (n bits per slot), the front as
// (slot << 32 | v) keys in rank order per slot, and the levels: one chunk per round and piece of (slot << 32 | v) keys, ascending,
// with the parent vertex and depth of each, merged so that their sizes at least halve from one chunk to the next.  od and the
// parent chains are binary searches over a side's O(log visited) chunks.
#include "edge_layers.cuh"

namespace b200 {

enum { SP_ACTIVE = 0, SP_FOUND = 1, SP_NULL = 2 };

struct SpOp { ECsr m, dp, dm; };
struct SpChunk { u64 off, n; };

// (slot, v)'s entry among a side's chunks: its position in lkey (and lval)
__device__ __forceinline__ bool sp_find(const SpChunk *__restrict__ ch, u32 nch, const u64 *__restrict__ lkey, u64 key, u64 *pos) {
    for (u32 c = 0; c < nch; c++) {
        const u64 a = lb64(lkey, ch[c].off, ch[c].off + ch[c].n, key);
        if (a < ch[c].off + ch[c].n && lkey[a] == key) { *pos = a; return true; }
    }
    return false;
}

// per active slot at the start of a round: Null when a front is empty or df + db >= max_hops, else the side to expand
__global__ void k_sp_begin(u64 S, u32 *__restrict__ state, const u64 *__restrict__ cnt, const u64 *__restrict__ depth, u64 max_hops,
                           u32 *__restrict__ side, u64 *__restrict__ nact) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        if (state[s] != SP_ACTIVE) continue;
        if (cnt[s] == 0 || cnt[S + s] == 0 || depth[s] + depth[S + s] >= max_hops) { state[s] = SP_NULL; continue; }
        side[s] = cnt[s] <= cnt[S + s] ? 0 : 1;
        atomicAdd((unsigned long long *)nact, 1ULL);
    }
}

// per front entry: its raw neighbour entries (every operand's m and dp row) when its slot expands this side, else 0; deg[nf] = 0
__global__ void k_sp_deg(const u64 *__restrict__ front, u64 nf, u32 sd, const u32 *__restrict__ state, const u32 *__restrict__ side,
                         const SpOp *__restrict__ ops, u32 nops, u64 *__restrict__ deg) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= nf; i += (u64)gridDim.x * blockDim.x) {
        u64 d = 0;
        if (i < nf) {
            const u64 s = front[i] >> 32, u = (u32)front[i];
            if (state[s] == SP_ACTIVE && side[s] == sd)
                for (u32 k = 0; k < nops; k++) {
                    if (ops[k].m.p) d += ops[k].m.p[u + 1] - ops[k].m.p[u];
                    if (ops[k].dp.p) d += ops[k].dp.p[u + 1] - ops[k].dp.p[u];
                }
        }
        deg[i] = d;
    }
}

// raw neighbour entry q of the piece (global position q0 + q): its front entry and neighbour, kept when the entry is effective (an
// m entry its own dm does not delete, or a dp entry) and the side has not seen the neighbour; key SLOT_NONE otherwise
__global__ void k_sp_emit(const u64 *__restrict__ front, const u64 *__restrict__ cum, u64 i0, u64 i1, u64 q0, u64 R,
                          const SpOp *__restrict__ ops, u32 nops, const u64 *__restrict__ vis, u64 nw, u64 *__restrict__ key,
                          u64 *__restrict__ val, u64 *__restrict__ nkept) {
    u64 kept = 0;
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < R; q += (u64)gridDim.x * blockDim.x) {
        const u64 g = q0 + q;
        const u64 a = i0 + list_at(cum + i0, i1 - i0, g);     // the last front entry with cum <= g
        const u64 s = front[a] >> 32, u = (u32)front[a];
        u64 o = g - cum[a];
        u32 v = 0;
        bool live = false;
        for (u32 k = 0; k < nops; k++) {
            const SpOp &op = ops[k];
            const u64 lm = op.m.p ? op.m.p[u + 1] - op.m.p[u] : 0;
            if (o < lm) { v = op.m.j[op.m.p[u] + o]; live = find_rc(op.dm, u, v) == ~0ULL; break; }
            o -= lm;
            const u64 ld = op.dp.p ? op.dp.p[u + 1] - op.dp.p[u] : 0;
            if (o < ld) { v = op.dp.j[op.dp.p[u] + o]; live = true; break; }
            o -= ld;
        }
        live = live && !slot_seen(vis, nw, s, v);
        key[q] = live ? (s << 32 | v) : SLOT_NONE;
        val[q] = a;
        kept += live;
    }
    if (kept) atomicAdd((unsigned long long *)nkept, (unsigned long long)kept);
}

// per distinct (slot, v) h: recorded in the side's new chunk with its parent, marked seen, and either a meet candidate (code = od,
// the piece's least od per slot in pod) or a survivor (code = SLOT_NONE, surv = 1)
__global__ void k_sp_classify(const u64 *__restrict__ key, const u64 *__restrict__ val, u64 E, const u32 *__restrict__ head,
                              const u64 *__restrict__ hpos, const u64 *__restrict__ front, u64 *__restrict__ vis_own,
                              const u64 *__restrict__ vis_oth, u64 nw, const SpChunk *__restrict__ och, u32 noch,
                              const u64 *__restrict__ olkey, const u64 *__restrict__ olval, const u64 *__restrict__ sdepth,
                              u64 *__restrict__ lkey, u64 *__restrict__ lval, u64 *__restrict__ code,
                              u32 *__restrict__ surv, u64 *__restrict__ pod) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x) {
        if (!head[e]) continue;
        const u64 h = hpos[e], k = key[e], s = k >> 32;
        const u32 v = (u32)k;
        lkey[h] = k;
        lval[h] = (u64)(u32)front[val[e]] << 32 | (u32)(sdepth[s] + 1);
        atomicOr((unsigned long long *)&vis_own[s * nw + (v >> 6)], 1ULL << (v & 63));
        u64 pos, od = SLOT_NONE;
        if (slot_seen(vis_oth, nw, s, v) && sp_find(och, noch, olkey, k, &pos)) {
            od = (u32)olval[pos];
            atomicMin((unsigned long long *)&pod[s], (unsigned long long)od);
            surv[h] = 0;
        } else {
            surv[h] = 1;
        }
        code[h] = od;
    }
}

// candidates at their slot's least od: the least (r, v) of the piece
__global__ void k_sp_tie(const u64 *__restrict__ lkey, const u64 *__restrict__ key, const u64 *__restrict__ val, u64 E,
                         const u32 *__restrict__ head, const u64 *__restrict__ hpos, const u64 *__restrict__ code,
                         const u64 *__restrict__ pod, u64 *__restrict__ prv) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x) {
        if (!head[e]) continue;
        const u64 h = hpos[e], s = key[e] >> 32;
        if (code[h] != SLOT_NONE && code[h] == pod[s]) atomicMin((unsigned long long *)&prv[s], (unsigned long long)(val[e] << 32 | (u32)lkey[h]));
    }
}

// a piece's meet replaces the round's only with a strictly smaller od (earlier pieces hold smaller ranks); the piece's cleared
__global__ void k_sp_merge(u64 S, u64 *__restrict__ pod, u64 *__restrict__ prv, u64 *__restrict__ bod, u64 *__restrict__ brv) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        if (pod[s] < bod[s]) { bod[s] = pod[s]; brv[s] = prv[s]; }
        pod[s] = SLOT_NONE; prv[s] = SLOT_NONE;
    }
}

// survivors, in (slot, v) order, as (parent rank, slot << 32 | v) for the re-sort by rank
__global__ void k_sp_survivors(const u64 *__restrict__ key, const u64 *__restrict__ val, u64 E, const u32 *__restrict__ head,
                               const u64 *__restrict__ hpos, const u32 *__restrict__ surv, const u64 *__restrict__ spos,
                               u64 *__restrict__ rk, u64 *__restrict__ nk) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x) {
        if (!head[e]) continue;
        const u64 h = hpos[e];
        if (!surv[h]) continue;
        rk[spos[h]] = val[e];
        nk[spos[h]] = key[e];
    }
}

// front entries of slots that stay active and do not expand side sd this round (their front carries over)
__global__ void k_sp_keep_flag(const u64 *__restrict__ front, u64 nf, u32 sd, const u32 *__restrict__ state,
                               const u32 *__restrict__ side, u32 *__restrict__ flag) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= nf; i += (u64)gridDim.x * blockDim.x) {
        u32 f = 0;
        if (i < nf) { const u64 s = front[i] >> 32; f = state[s] == SP_ACTIVE && side[s] != sd; }
        flag[i] = f;
    }
}

// the end of a round: the expanded side one level deeper; a slot with a meet is found
__global__ void k_sp_end(u64 S, u32 *__restrict__ state, const u32 *__restrict__ side, u64 *__restrict__ depth,
                         const u64 *__restrict__ brv) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        if (state[s] != SP_ACTIVE) continue;
        depth[side[s] * S + s]++;
        if (brv[s] != SLOT_NONE) state[s] = SP_FOUND;
    }
}

// per slot its front entries; one atomic per run of equal slots in a warp (a front is mostly grouped by slot)
__global__ void k_sp_count(const u64 *__restrict__ front, u64 nf, u64 *__restrict__ cnt) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 s = i < nf ? front[i] >> 32 : SLOT_NONE;
    const unsigned peers = __match_any_sync(0xffffffffu, s);
    if (i < nf && (u32)(__ffs(peers) - 1) == (threadIdx.x & 31)) atomicAdd((unsigned long long *)&cnt[s], (unsigned long long)__popc(peers));
}

// per found slot: nodes on its path, depth_F(meet) + depth_B(meet) + 1; 0 otherwise.  lval: parent << 32 | depth
struct SpSide { const SpChunk *ch; u32 nch; const u64 *lkey, *lval; };
__global__ void k_sp_len(u64 S, const u32 *__restrict__ state, const u64 *__restrict__ brv, SpSide F, SpSide B, u64 *__restrict__ len) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        u64 l = 0;
        if (state[s] == SP_FOUND) {
            const u64 k = s << 32 | (u32)brv[s];
            u64 pf = 0, pb = 0;
            sp_find(F.ch, F.nch, F.lkey, k, &pf);
            sp_find(B.ch, B.nch, B.lkey, k, &pb);
            l = (u64)(u32)F.lval[pf] + (u32)B.lval[pb] + 1;
        }
        len[s] = l;
    }
}
// the path from src to dst: forward parents from the meet down to src, then backward parents down to dst
__global__ void k_sp_write(u64 S, const u32 *__restrict__ state, const u64 *__restrict__ brv, SpSide F, SpSide B,
                           const u64 *__restrict__ off, u32 *__restrict__ out) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        if (state[s] != SP_FOUND) continue;
        const u32 m = (u32)brv[s];
        u64 pos = 0;
        sp_find(F.ch, F.nch, F.lkey, s << 32 | m, &pos);
        const u64 df = (u32)F.lval[pos];
        u32 *o = out + off[s];
        o[df] = m;
        u32 cur = m;
        for (u64 i = df; i > 0; i--) {
            sp_find(F.ch, F.nch, F.lkey, s << 32 | cur, &pos);
            cur = (u32)(F.lval[pos] >> 32);
            o[i - 1] = cur;
        }
        sp_find(B.ch, B.nch, B.lkey, s << 32 | m, &pos);
        const u64 db = (u32)B.lval[pos];
        cur = m;
        for (u64 i = 1; i <= db; i++) {
            sp_find(B.ch, B.nch, B.lkey, s << 32 | cur, &pos);
            cur = (u32)(B.lval[pos] >> 32);
            o[df + i] = cur;
        }
    }
}

// the seeds: front, depth-0 chunk and visited bit per slot (src on F, dst on B)
__global__ void k_sp_seed(const u64 *__restrict__ ends, u64 S, u64 nw, u64 *__restrict__ front, u64 *__restrict__ lkey,
                          u64 *__restrict__ lval, u64 *__restrict__ vis) {
    for (u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (u64)gridDim.x * blockDim.x) {
        const u32 v = (u32)ends[s];
        front[s] = lkey[s] = s << 32 | v;
        lval[s] = (u64)v << 32;
        vis[s * nw + (v >> 6)] |= 1ULL << (v & 63);
    }
}

// ---- host side ----

struct SpSideState {
    DevBuf<u64> vis, front, lkey, lval;
    u64 nf = 0, nl = 0;
    std::vector<SpChunk> chunks;
    DevBuf<SpChunk> dch;                       // chunks on the device, refreshed by upload()
    DevBuf<SpOp> ops;
    u32 nops = 0;
    void upload() {
        dch.alloc(chunks.size());
        h2d(dch.ptr, chunks.data(), chunks.size());
    }
    SpSide view() const { return SpSide{dch.ptr, (u32)chunks.size(), lkey.ptr, lval.ptr}; }
    // Level chunks kept in sizes that at least halve from one to the next: the newest chunk is merged into the one before while
    // that one is at most twice its size.  Keys are unique within a side, so a merge is a sort of the two adjacent chunks.  A
    // lookup then searches at most log2(visited) + 1 chunks, and each entry is re-sorted O(log) times.
    void merge_tail() {
        while (chunks.size() >= 2) {
            SpChunk &a = chunks[chunks.size() - 2];
            const SpChunk b = chunks.back();
            if (a.n > 2 * b.n) break;
            sort_pairs_u64(lkey.ptr + a.off, lval.ptr + a.off, a.n + b.n, SLOT_KEY_BITS);
            a.n += b.n;
            chunks.pop_back();
        }
    }
};

// One side's expansion for the slots that chose it this round.  Returns the raw neighbour entries scanned.
static u64 sp_expand(SpSideState &own, SpSideState &oth, u32 sd, u64 S, u64 nw, DevBuf<u32> &state, DevBuf<u32> &side,
                     const DevBuf<u64> &depth, DevBuf<u64> &pod, DevBuf<u64> &prv, DevBuf<u64> &bod, DevBuf<u64> &brv, u64 budget) {
    const u64 nf = own.nf;
    // the front entries that carry over
    DevBuf<u32> kf(nf + 1);
    DevBuf<u64> kpos(nf + 1);
    LAUNCH(k_sp_keep_flag, grid_for(nf + 1, PAIR_T), PAIR_T, 0, own.front.ptr, nf, sd, state.ptr, side.ptr, kf.ptr);
    exclusive_scan_u32_to_u64(kf.ptr, kpos.ptr, nf + 1);
    const u64 nkeep = read_scalar(kpos.ptr + nf);
    DevBuf<u64> next(std::max<u64>(nkeep, 1));
    if (nkeep) scatter_flagged(own.front.ptr, nf, kf.ptr, kpos.ptr, next.ptr);
    u64 nnext = nkeep;
    kf.release(); kpos.release();

    DevBuf<u64> cum(nf + 1);
    LAUNCH(k_sp_deg, grid_for(nf + 1, PAIR_T), PAIR_T, 0, own.front.ptr, nf, sd, state.ptr, side.ptr, own.ops.ptr, own.nops, cum.ptr);
    exclusive_scan_u64(cum.ptr, cum.ptr, nf + 1);
    const u64 total = nf ? read_scalar(cum.ptr + nf) : 0;
    DevBuf<u64> scal(1);
    oth.upload();
    for_each_piece(cum.ptr, nf, total, budget, [&](u64 i0, u64 i1, u64 q0, u64 q1) {
        const u64 R = q1 - q0;
        DevBuf<u64> key(R), val(R);
        CUDA_TRY(cudaMemsetAsync(scal.ptr, 0, sizeof(u64), stream()));
        LAUNCH(k_sp_emit, grid_for(R, PAIR_T, 8 * (u64)ctx().num_sms), PAIR_T, 0, own.front.ptr, cum.ptr, i0, i1, q0, R, own.ops.ptr,
               own.nops, own.vis.ptr, nw, key.ptr, val.ptr, scal.ptr);
        const u64 E = read_scalar(scal.ptr);
        if (!E) return;
        sort_pairs_u64(key.ptr, val.ptr, R, SLOT_KEY_BITS);            // stable: the least rank leads each (slot, v)
        DevBuf<u32> head(E + 1);
        DevBuf<u64> hpos(E + 1);
        const u64 nh = run_heads(key.ptr, E, head.ptr, hpos.ptr);
        grow(own.lkey, own.nl, own.nl + nh);
        grow(own.lval, own.nl, own.nl + nh);
        DevBuf<u64> code(nh), spos(nh + 1);
        DevBuf<u32> surv(nh + 1);
        CUDA_TRY(cudaMemsetAsync(surv.ptr + nh, 0, sizeof(u32), stream()));
        LAUNCH(k_sp_classify, grid_for(E, PAIR_T), PAIR_T, 0, key.ptr, val.ptr, E, head.ptr, hpos.ptr, own.front.ptr, own.vis.ptr,
               oth.vis.ptr, nw, oth.dch.ptr, (u32)oth.chunks.size(), oth.lkey.ptr, oth.lval.ptr, depth.ptr + sd * S,
               own.lkey.ptr + own.nl, own.lval.ptr + own.nl, code.ptr, surv.ptr, pod.ptr);
        own.chunks.push_back(SpChunk{own.nl, nh});
        own.nl += nh;
        LAUNCH(k_sp_tie, grid_for(E, PAIR_T), PAIR_T, 0, own.lkey.ptr + own.nl - nh, key.ptr, val.ptr, E, head.ptr, hpos.ptr, code.ptr,
               pod.ptr, prv.ptr);
        LAUNCH(k_sp_merge, grid_for(S, PAIR_T), PAIR_T, 0, S, pod.ptr, prv.ptr, bod.ptr, brv.ptr);
        own.merge_tail();                                       // after k_sp_tie, which reads the new chunk in place
        exclusive_scan_u32_to_u64(surv.ptr, spos.ptr, nh + 1);
        const u64 ns = read_scalar(spos.ptr + nh);
        if (!ns) return;
        DevBuf<u64> rk(ns), nk(ns);
        LAUNCH(k_sp_survivors, grid_for(E, PAIR_T), PAIR_T, 0, key.ptr, val.ptr, E, head.ptr, hpos.ptr, surv.ptr, spos.ptr, rk.ptr,
               nk.ptr);
        sort_pairs_u64(rk.ptr, nk.ptr, ns, bit_length(nf));          // stable: (rank, v)
        grow(next, nnext, nnext + ns);
        d2d(next.ptr + nnext, nk.ptr, ns);
        nnext += ns;
    });
    own.front = std::move(next);
    own.nf = nnext;
    return total;
}

u64 shortest_path(const u64 *h_src, const u64 *h_dst, u64 np, const std::vector<SpOperand> &fwd, const std::vector<SpOperand> &bwd,
                  u64 n, u64 max_hops, u64 budget, std::vector<u64> &len, std::vector<u32> &nodes) {
    TimedScope ts(TK_SHORTEST_PATH, 0);
    const u64 nw = (n + 63) / 64;
    size_t fr = 0, tot = 0;
    CUDA_TRY(cudaMemGetInfo(&fr, &tot));
    budget = piece_budget(budget, fr);
    // the two visited bitmaps of a slice take at most a quarter of the free memory
    const u64 per_slot = 2 * nw * 8;
    const u64 S_max = std::max<u64>(1, std::min<u64>(1024, fr / 4 / per_slot));
    len.assign(np, 0);
    nodes.clear();
    u64 flops = 0;
    auto make_ops = [](const std::vector<SpOperand> &v, SpSideState &st) {
        std::vector<SpOp> h(v.size());
        for (size_t k = 0; k < v.size(); k++) h[k] = SpOp{ecsr(v[k].m), ecsr(v[k].dp), ecsr(v[k].dm)};
        st.ops.alloc(h.size());
        h2d(st.ops.ptr, h.data(), h.size());
        st.nops = (u32)h.size();
    };
    auto run_slice = [&](u64 p0, u64 S) {
        SpSideState side_st[2];
        make_ops(fwd, side_st[0]);
        make_ops(bwd, side_st[1]);
        DevBuf<u64> ends(S);
        for (int sd = 0; sd < 2; sd++) {
            SpSideState &st = side_st[sd];
            h2d(ends.ptr, (sd ? h_dst : h_src) + p0, S);
            st.vis.alloc(S * nw);
            st.vis.zero();
            st.front.alloc(S); st.lkey.alloc(S); st.lval.alloc(S);
            LAUNCH(k_sp_seed, grid_for(S, PAIR_T), PAIR_T, 0, ends.ptr, S, nw, st.front.ptr, st.lkey.ptr, st.lval.ptr, st.vis.ptr);
            st.nf = st.nl = S;
            st.chunks = {SpChunk{0, S}};
        }
        DevBuf<u32> state(S), side(S);
        DevBuf<u64> cnt(2 * S), depth(2 * S), pod(S), prv(S), bod(S), brv(S), scal(1);
        state.zero(); side.zero(); depth.zero();
        CUDA_TRY(cudaMemsetAsync(pod.ptr, 0xff, S * 8, stream()));
        CUDA_TRY(cudaMemsetAsync(prv.ptr, 0xff, S * 8, stream()));
        CUDA_TRY(cudaMemsetAsync(bod.ptr, 0xff, S * 8, stream()));
        CUDA_TRY(cudaMemsetAsync(brv.ptr, 0xff, S * 8, stream()));
        while (true) {
            cnt.zero();
            for (int sd = 0; sd < 2; sd++)
                if (side_st[sd].nf) LAUNCH(k_sp_count, grid_for(side_st[sd].nf, PAIR_T), PAIR_T, 0, side_st[sd].front.ptr, side_st[sd].nf,
                                           cnt.ptr + sd * S);
            CUDA_TRY(cudaMemsetAsync(scal.ptr, 0, 8, stream()));
            LAUNCH(k_sp_begin, grid_for(S, PAIR_T), PAIR_T, 0, S, state.ptr, cnt.ptr, depth.ptr, max_hops, side.ptr, scal.ptr);
            if (!read_scalar(scal.ptr)) break;
            for (int sd = 0; sd < 2; sd++) {
                SpSideState &own = side_st[sd];
                if (own.nf >= ((u64)1 << 32)) throw GrbError(-8, "shortest_path: a front of 2^32 entries");   // ranks are 32 bits
                flops += sp_expand(own, side_st[1 - sd], (u32)sd, S, nw, state, side, depth, pod, prv, bod, brv, budget);
            }
            LAUNCH(k_sp_end, grid_for(S, PAIR_T), PAIR_T, 0, S, state.ptr, side.ptr, depth.ptr, brv.ptr);
        }
        // paths
        for (int sd = 0; sd < 2; sd++) side_st[sd].upload();
        DevBuf<u64> dl(S + 1), off(S + 1);
        LAUNCH(k_sp_len, grid_for(S, PAIR_T), PAIR_T, 0, S, state.ptr, brv.ptr, side_st[0].view(), side_st[1].view(), dl.ptr);
        d2h(len.data() + p0, dl.ptr, S);
        sync_stream();
        std::vector<u64> hoff(S + 1, 0);
        for (u64 s = 0; s < S; s++) hoff[s + 1] = hoff[s] + len[p0 + s];
        if (hoff[S]) {
            h2d(off.ptr, hoff.data(), S + 1);
            DevBuf<u32> out(hoff[S]);
            LAUNCH(k_sp_write, grid_for(S, PAIR_T), PAIR_T, 0, S, state.ptr, brv.ptr, side_st[0].view(), side_st[1].view(), off.ptr, out.ptr);
            const size_t base = nodes.size();                   // no allocation after this: a retried slice appends nothing
            nodes.resize(base + hoff[S]);
            d2h(nodes.data() + base, out.ptr, hoff[S]);
            sync_stream();
        }
    };
    // the bitmaps size a slice up front; the fronts and level entries grow with what each pair visits
    for_each_slice(np, S_max, run_slice);
    return flops;
}

} // namespace b200
