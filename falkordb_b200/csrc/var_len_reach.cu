// var_len_reach.cu -- the start's own entry of a bidirectional variable-length reach (B200_var_len_reach_both).
//
// G' is the undirected multigraph with one edge per live relationship of the types.  A reach over the union of every type's
// forward and transpose layers (graph_api.cu) is exact for every v != s: a shortest walk is a path, and a path is a trail.  It is
// wrong for s itself, which a trail of 1..k edges reaches iff G' holds a cycle through s of length g(s) <= k (a closed trail
// shortcuts to a cycle through s that is no longer and uses a subset of its edges).  This file decides g(s) <= k:
//   g = 1, 2  the starts' adjacency under Both (edge_adjacency: one entry per live relationship, a self-loop once) sorted by
//             (slot, neighbour): a run whose neighbour is s is a self-loop, a run of two or more is two relationships to one c.
//   g >= 3    s - c - ... - c' - s with c != c', the middle a path of g - 2 edges in G' - s.  The distinct neighbours c != s get
//             ranks r(c) in 0 .. d_s; two distinct ranks differ in some bit b < ceil(log2 d_s).  Row (s, b) of a frontier starts
//             from X0 = {c : bit b of r(c) = 0} with X0 u {s} reached (so no walk passes through s) and aims at
//             T = {c : bit b of r(c) = 1}; k - 2 masked levels (graph_api.cu's reach_hop) find T iff g(s) <= k.  A hit decides the
//             slot and drops every row of it from the frontier.
// Rows go in chunks of at most 1024 (the frontier form's limit); the host reads a handful of words per chunk and level.
#include "edge_layers.cuh"

namespace b200 {

static const u32 NO_ROW = ~0u;

// per adjacency entry: (slot << 32) | neighbour
__global__ void k_vb_keys(const u64 *__restrict__ adj_p, u64 nu, const u32 *__restrict__ node, u64 E, u64 *__restrict__ key) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x)
        key[e] = (list_at(adj_p, nu, e) << 32) | node[e];
}
// the runs of the sorted keys: flag bit 0 a self-loop (g = 1), bit 1 two relationships to one neighbour (g = 2); nh[e] = 1 at the
// head of a run whose neighbour is not the start
__global__ void k_vb_runs(const u64 *__restrict__ key, u64 E, const u64 *__restrict__ u, u32 *__restrict__ flag, u32 *__restrict__ nh) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x) {
        const u64 k = key[e], j = k >> 32, c = k & 0xffffffffULL;
        const bool head = e == 0 || key[e - 1] != k;
        u32 h = 0;
        if (head) {
            if (c == u[j]) atomicOr(&flag[j], 1u);
            else {
                h = 1;
                if (e + 1 < E && key[e + 1] == k) atomicOr(&flag[j], 2u);
            }
        }
        nh[e] = h;
    }
}
// the distinct neighbours c != s, slot-major and ascending within a slot: their rank is their position minus the slot's base
__global__ void k_vb_neigh(const u64 *__restrict__ key, u64 E, const u32 *__restrict__ nh, const u64 *__restrict__ npos,
                           u32 *__restrict__ dn, u32 *__restrict__ dslot) {
    for (u64 e = (u64)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (u64)gridDim.x * blockDim.x)
        if (nh[e]) { dn[npos[e]] = (u32)key[e]; dslot[npos[e]] = (u32)(key[e] >> 32); }
}
// per slot j <= nu: nbase[j] = its first distinct neighbour; dec[j] = decided by g <= 2 (or no closure needed); nrow[j] = its
// bit-split rows
__global__ void k_vb_slots(const u64 *__restrict__ adj_p, u64 nu, const u64 *__restrict__ npos, const u32 *__restrict__ flag,
                           u64 max_hops, u64 *__restrict__ nbase, u32 *__restrict__ dec, u64 *__restrict__ nrow) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j <= nu; j += (u64)gridDim.x * blockDim.x) {
        nbase[j] = npos[adj_p[j]];
        if (j == nu) { nrow[j] = 0; continue; }
        const u64 d = npos[adj_p[j + 1]] - npos[adj_p[j]];
        const u32 f = flag[j];
        const bool in = ((f & 1) && max_hops >= 1) || ((f & 2) && max_hops >= 2);
        dec[j] = in ? 1 : 0;
        nrow[j] = !in && max_hops >= 3 && d >= 2 ? 64 - __clzll((long long)(d - 1)) : 0;
    }
}
// the distinct-neighbour range of the rows [r0, r1)
__global__ void k_vb_range(const u64 *__restrict__ rowbase, const u64 *__restrict__ nbase, u64 nu, u64 r0, u64 r1, u64 *__restrict__ q) {
    q[0] = nbase[list_at(rowbase, nu, r0)];
    q[1] = nbase[list_at(rowbase, nu, r1 - 1) + 1];
}

struct VbRows { const u64 *rowbase, *nbase; const u32 *dn, *dslot; u64 r0, r1; u32 W; };

// the local row of bit b of slot j, or NO_ROW outside the chunk
__device__ __forceinline__ u32 local_row(const VbRows &A, u64 j, u32 b) {
    const u64 r = A.rowbase[j] + b;
    return r >= A.r0 && r < A.r1 ? (u32)(r - A.r0) : NO_ROW;
}

// seeds: F = X0, R = X0 per row (the starts are added by k_vb_seed_start).  A slot decided in an earlier chunk (its rows straddle
// the boundary) is not seeded: its rows stay empty.
__global__ void k_vb_seed(VbRows A, u64 q0, u64 q1, const u32 *__restrict__ dec, u64 *__restrict__ F, u64 *__restrict__ R) {
    for (u64 q = q0 + (u64)blockIdx.x * blockDim.x + threadIdx.x; q < q1; q += (u64)gridDim.x * blockDim.x) {
        const u64 j = A.dslot[q];
        if (dec[j]) continue;
        const u64 c = A.dn[q], rank = q - A.nbase[j];
        const u32 nb = (u32)(A.rowbase[j + 1] - A.rowbase[j]);
        for (u32 b = 0; b < nb; b++) {
            const u32 lr = local_row(A, j, b);
            if (lr == NO_ROW || ((rank >> b) & 1)) continue;
            const u64 w = c * A.W + (lr >> 6), bit = 1ULL << (lr & 63);
            atomicOr((unsigned long long *)&F[w], (unsigned long long)bit);
            atomicOr((unsigned long long *)&R[w], (unsigned long long)bit);
        }
    }
}
__global__ void k_vb_seed_start(VbRows A, u64 nu, const u64 *__restrict__ u, u64 *__restrict__ R) {
    for (u64 lr = (u64)blockIdx.x * blockDim.x + threadIdx.x; lr < A.r1 - A.r0; lr += (u64)gridDim.x * blockDim.x) {
        const u64 s = u[list_at(A.rowbase, nu, A.r0 + lr)];
        atomicOr((unsigned long long *)&R[s * A.W + (lr >> 6)], (unsigned long long)(1ULL << (lr & 63)));
    }
}
// a target in a row's new frontier decides the row's slot
__global__ void k_vb_hit(VbRows A, u64 q0, u64 q1, const u64 *__restrict__ F, u32 *__restrict__ dec) {
    for (u64 q = q0 + (u64)blockIdx.x * blockDim.x + threadIdx.x; q < q1; q += (u64)gridDim.x * blockDim.x) {
        const u64 j = A.dslot[q], c = A.dn[q], rank = q - A.nbase[j];
        const u32 nb = (u32)(A.rowbase[j + 1] - A.rowbase[j]);
        for (u32 b = 0; b < nb; b++) {
            const u32 lr = local_row(A, j, b);
            if (lr == NO_ROW || !((rank >> b) & 1)) continue;
            if ((F[c * A.W + (lr >> 6)] >> (lr & 63)) & 1) { dec[j] = 1; break; }
        }
    }
}
// the rows of decided slots, as a W-word row mask
__global__ void k_vb_drop(VbRows A, u64 nu, const u32 *__restrict__ dec, u64 *__restrict__ drop) {
    for (u64 lr = (u64)blockIdx.x * blockDim.x + threadIdx.x; lr < A.r1 - A.r0; lr += (u64)gridDim.x * blockDim.x)
        if (dec[list_at(A.rowbase, nu, A.r0 + lr)])
            atomicOr((unsigned long long *)&drop[lr >> 6], (unsigned long long)(1ULL << (lr & 63)));
}
// F &= ~drop per row; live[w] = the rows with a frontier left.  The grid stride is a multiple of W (a power of two <= 16), so a
// thread always reads the same word slot of its vertices and the lanes of one slot meet in a butterfly.
__global__ void k_vb_mask(u64 *__restrict__ F, u64 words, u32 W, const u64 *__restrict__ drop, u64 *__restrict__ live) {
    const u32 w = threadIdx.x & (W - 1);
    const u64 d = ~drop[w];
    u64 acc = 0;
    for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < words; t += (u64)gridDim.x * blockDim.x) {
        const u64 x = F[t], y = x & d;
        if (y != x) F[t] = y;
        acc |= y;
    }
    for (u32 o = 16; o >= W; o >>= 1) acc |= __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) < W && acc) atomicOr((unsigned long long *)&live[w], (unsigned long long)acc);
}
__global__ void k_vb_count(const u64 *__restrict__ live, u32 W, u64 *__restrict__ n) {
    u64 c = 0;
    for (u32 w = 0; w < W; w++) c += __popcll(live[w]);
    *n = c;
}

// the fix-up of row i: (i, starts[i]) kept iff the start is decided
__global__ void k_vb_fix_bits(const u64 *__restrict__ s, u64 n, const u32 *__restrict__ slot, const u32 *__restrict__ dec, u32 W,
                              u64 *__restrict__ R) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        if (!dec[slot[i]]) atomicAnd((unsigned long long *)&R[s[i] * W + (i >> 6)], ~(unsigned long long)(1ULL << (i & 63)));
}
// CSR form: drop[i] = row i loses its start; len[i] = its new length (len[n] = 0)
__global__ void k_vb_fix_len(const u64 *__restrict__ s, u64 n, const u32 *__restrict__ slot, const u32 *__restrict__ dec,
                             const u64 *__restrict__ p, const u32 *__restrict__ j, u32 *__restrict__ drop, u64 *__restrict__ len) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += (u64)gridDim.x * blockDim.x) {
        if (i == n) { len[n] = 0; continue; }
        const u64 a = p[i], e = p[i + 1], q = lb32(j, a, e, (u32)s[i]);
        const u32 d = !dec[slot[i]] && q < e && j[q] == (u32)s[i] ? 1 : 0;
        drop[i] = d;
        len[i] = e - a - d;
    }
}
__global__ void k_vb_fix_copy(const u64 *__restrict__ s, u64 n, const u32 *__restrict__ drop, const u64 *__restrict__ p,
                              const u32 *__restrict__ j, u64 nnz, const u64 *__restrict__ op, u32 *__restrict__ oj) {
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < nnz; q += (u64)gridDim.x * blockDim.x) {
        const u64 i = list_at(p, n, q);
        const u32 c = j[q], x = (u32)s[i];
        if (drop[i] && c == x) continue;
        oj[op[i] + (q - p[i]) - (drop[i] && c > x ? 1 : 0)] = c;
    }
}

void vlb_plan(const u64 *h_starts, u64 nstarts, const std::vector<EdgeTypeDev> &types, u64 max_hops, VlbPlan &P) {
    const u32 grid = (u32)ctx().num_sms * 8;
    const ETypes ty(types);
    // Compulsory bytes ("var_len_reach_both"), this pass: 24 per start (its id, twice for the sort, and its slot), the adjacency
    // fetch (edge_expand's formula), 28 per adjacency entry (the key written, read by the sort and the run pass, its head flag and
    // scan), 8 per distinct neighbour (vertex and slot), 40 per distinct start (flags, bases, decision)
    TimedScope ts(TK_VAR_LEN_REACH_BOTH, 0);
    u64 bytes = 24 * nstarts;
    P.n = nstarts;
    P.ds.alloc(nstarts);
    h2d(P.ds.ptr, h_starts, nstarts);
    P.u.alloc(nstarts);
    d2d(P.u.ptr, P.ds.ptr, nstarts);
    const u64 nu = P.nu = unique_sorted(P.u, nstarts, 32);
    P.slot.alloc(nstarts);
    node_rows(P.ds.ptr, nstarts, P.u.ptr, nu, nullptr, P.slot.ptr, nullptr);
    DevBuf<u64> adj_p, adj_edge;
    DevBuf<u32> adj_node;
    const u64 E = edge_adjacency(ty, P.u.ptr, nu, 2, adj_p, adj_node, adj_edge, &bytes);
    adj_edge.release();
    DevBuf<u64> key(E), npos(E + 1);
    DevBuf<u32> flag(nu), nh(E + 1);
    flag.zero();
    CUDA_TRY(cudaMemsetAsync(nh.ptr + E, 0, sizeof(u32), stream()));
    if (E) {
        LAUNCH(k_vb_keys, grid_for(E, 256, grid), 256, 0, adj_p.ptr, nu, adj_node.ptr, E, key.ptr);
        adj_node.release();
        sort_keys_u64(key.ptr, E, 32 + bit_length(nu));
        LAUNCH(k_vb_runs, grid_for(E, 256, grid), 256, 0, key.ptr, E, P.u.ptr, flag.ptr, nh.ptr);
    }
    exclusive_scan_u32_to_u64(nh.ptr, npos.ptr, E + 1);
    P.Q = read_scalar(npos.ptr + E);
    P.dn.alloc(P.Q); P.dslot.alloc(P.Q);
    if (E) LAUNCH(k_vb_neigh, grid_for(E, 256, grid), 256, 0, key.ptr, E, nh.ptr, npos.ptr, P.dn.ptr, P.dslot.ptr);
    P.nbase.alloc(nu + 1); P.rowbase.alloc(nu + 1); P.dec.alloc(nu);
    DevBuf<u64> nrow(nu + 1);
    LAUNCH(k_vb_slots, grid_for(nu + 1, 256, grid), 256, 0, adj_p.ptr, nu, npos.ptr, flag.ptr, max_hops, P.nbase.ptr, P.dec.ptr,
           nrow.ptr);
    exclusive_scan_u64(nrow.ptr, P.rowbase.ptr, nu + 1);
    P.rows = read_scalar(P.rowbase.ptr + nu);
    ts.bytes = bytes + 28 * E + 8 * P.Q + 40 * nu;
}

static VbRows rows_of(const VlbPlan &P, u64 r0, u64 r1, u32 W) {
    return VbRows{P.rowbase.ptr, P.nbase.ptr, P.dn.ptr, P.dslot.ptr, r0, r1, W};
}

static void new_bits(DevBits &X, u64 rows, u64 n, u32 W) {
    X.clear();
    X.nrows = rows; X.ncols = n; X.W = W;
    X.w.alloc(n * W);
    X.w.zero();
}

void vlb_seed(VlbPlan &P, u64 r0, u64 r1, u64 n, DevBits &F, DevBits &R) {
    const u32 grid = (u32)ctx().num_sms * 8, W = bits_words_for(r1 - r0);
    // Compulsory bytes: F and R written whole (16 n W), 16 per distinct neighbour of the chunk (vertex, slot, two bases)
    TimedScope ts(TK_VAR_LEN_REACH_BOTH, 0);
    new_bits(F, r1 - r0, n, W);
    new_bits(R, r1 - r0, n, W);
    DevBuf<u64> q(2);
    LAUNCH(k_vb_range, 1, 1, 0, P.rowbase.ptr, P.nbase.ptr, P.nu, r0, r1, q.ptr);
    P.q0 = read_scalar(q.ptr);
    P.q1 = read_scalar(q.ptr + 1);
    const VbRows A = rows_of(P, r0, r1, W);
    if (P.q1 > P.q0) LAUNCH(k_vb_seed, grid_for(P.q1 - P.q0, 256, grid), 256, 0, A, P.q0, P.q1, P.dec.ptr, F.w.ptr, R.w.ptr);
    LAUNCH(k_vb_seed_start, grid_for(r1 - r0, 256, grid), 256, 0, A, P.nu, P.u.ptr, R.w.ptr);
    ts.bytes = 16 * n * W + 16 * (P.q1 - P.q0);
}

u64 vlb_level(VlbPlan &P, u64 r0, u64 r1, DevBits &F) {
    const u32 grid = (u32)ctx().num_sms * 8, W = F.W;
    // Compulsory bytes: 24 per distinct neighbour of the chunk (vertex, slot, two bases, the frontier word), F read whole (8 n W)
    TimedScope ts(TK_VAR_LEN_REACH_BOTH, 24 * (P.q1 - P.q0) + 8 * F.ncols * W);
    const VbRows A = rows_of(P, r0, r1, W);
    if (P.q1 > P.q0) LAUNCH(k_vb_hit, grid_for(P.q1 - P.q0, 256, grid), 256, 0, A, P.q0, P.q1, F.w.ptr, P.dec.ptr);
    DevBuf<u64> drop(W), live(W), cnt(1);
    drop.zero(); live.zero();
    LAUNCH(k_vb_drop, grid_for(r1 - r0, 256, grid), 256, 0, A, P.nu, P.dec.ptr, drop.ptr);
    const u64 words = F.ncols * W;
    if (words) LAUNCH(k_vb_mask, grid_for(words, 256, (u64)ctx().num_sms * 16), 256, 0, F.w.ptr, words, W, drop.ptr, live.ptr);
    LAUNCH(k_vb_count, 1, 1, 0, live.ptr, W, cnt.ptr);
    return read_scalar(cnt.ptr);
}

void vlb_fix_bits(const VlbPlan &P, DevBits &R) {
    // Compulsory bytes: 24 per start (id, slot, decision, the word it clears)
    TimedScope ts(TK_VAR_LEN_REACH_BOTH, 24 * P.n);
    LAUNCH(k_vb_fix_bits, grid_for(P.n, 256, (u32)ctx().num_sms * 8), 256, 0, P.ds.ptr, P.n, P.slot.ptr, P.dec.ptr, R.W, R.w.ptr);
}

void vlb_fix_csr(const VlbPlan &P, const DevCSR &R, DevCSR &out) {
    const u32 grid = (u32)ctx().num_sms * 8;
    const u64 n = P.n;
    // Compulsory bytes: 40 per row (id, slot, decision, row pointers, new length), 8 per entry (read and written)
    TimedScope ts(TK_VAR_LEN_REACH_BOTH, 40 * n + 8 * R.nnz);
    DevBuf<u32> drop(n);
    DevBuf<u64> len(n + 1);
    out.nrows = R.nrows; out.ncols = R.ncols;
    out.p.alloc(n + 1);
    LAUNCH(k_vb_fix_len, grid_for(n + 1, 256, grid), 256, 0, P.ds.ptr, n, P.slot.ptr, P.dec.ptr, R.p.ptr, R.j.ptr, drop.ptr, len.ptr);
    exclusive_scan_u64(len.ptr, out.p.ptr, n + 1);
    out.nnz = read_scalar(out.p.ptr + n);
    out.j.alloc(out.nnz);
    if (R.nnz) LAUNCH(k_vb_fix_copy, grid_for(R.nnz, 256, grid), 256, 0, P.ds.ptr, n, drop.ptr, R.p.ptr, R.j.ptr, R.nnz, out.p.ptr, out.j.ptr);
}

} // namespace b200
