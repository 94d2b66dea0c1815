// edge_layers.cuh -- a relationship Tensor's live layers as the device reads them, and the point lookups over them that both
// B200_expand_edges (edges.cu) and the write plans (writes.cu) make: find_rc, Tensor::eff_get, and a multi-edge pair's merged id
// list (me \ me_dm) u me_dp.  Also the plumbing the relationship searches share: the per-level adjacency fetch of a key list
// (NodeAdj), and the slices, pieces and slot keys of the batched pair searches (shortest_path.cu, all_shortest_paths.cu).
#pragma once
#include "common.cuh"
#include "ops.cuh"
#include <algorithm>
#include <functional>

namespace b200 {

static const u64 EE_MULTI = ~0ULL;   // Tensor's MULTI_EDGE value (tensor.rs:206)

struct ECsr { const u64 *p; const u32 *j; const u64 *x; };          // p null: the layer is absent
struct EStore { const u64 *key; const u64 *ptr; const u64 *id; u64 nkey; };
struct EType { ECsr m, dp, dm, mt, mtdp, mtdm; EStore me, medp, medm; };

static ECsr ecsr(const DevCSR *A) {
    if (!A || !A->nnz) return ECsr{nullptr, nullptr, nullptr};
    return ECsr{A->p.ptr, A->j.ptr, A->x.ptr};
}
static EStore estore(const DevIdStore *S) {
    if (!S || !S->nkey) return EStore{nullptr, nullptr, nullptr, 0};
    return EStore{S->key.ptr, S->ptr.ptr, S->id.ptr, S->nkey};
}
static EType etype(const EdgeTypeDev &x) {
    return EType{ecsr(x.m), ecsr(x.dp), ecsr(x.dm), ecsr(x.mt), ecsr(x.mt_dp), ecsr(x.mt_dm), estore(x.me), estore(x.me_dp),
                 estore(x.me_dm)};
}
// the types of a call, uploaded: d[0 .. T)
struct ETypes {
    DevBuf<EType> d;
    u32 T;
    explicit ETypes(const std::vector<EdgeTypeDev> &types);   // edges.cu
};

// largest g with lstart[g] <= e (lstart ascending, lstart[0] = 0): the segment of flat position e behind a scan of lengths
__device__ __forceinline__ u64 list_at(const u64 *__restrict__ lstart, u64 G, u64 e) { return last_le(lstart, 0, G - 1, e); }
// position of (r, c) in A, or ~0
__device__ __forceinline__ u64 find_rc(const ECsr &A, u64 r, u32 c) {
    if (!A.p) return ~0ULL;
    const u64 e = A.p[r + 1], q = lb32(A.j, A.p[r], e, c);
    return q < e && A.j[q] == c ? q : ~0ULL;
}
// Tensor::eff_get (tensor.rs:290-303): dp if present, else nothing if dm holds it, else m
__device__ __forceinline__ bool eff_get(const EType &t, u64 r, u32 c, u64 *v) {
    u64 q = find_rc(t.dp, r, c);
    if (q != ~0ULL) { *v = t.dp.x[q]; return true; }
    if (find_rc(t.dm, r, c) != ~0ULL) return false;
    q = find_rc(t.m, r, c);
    if (q == ~0ULL) return false;
    *v = t.m.x[q];
    return true;
}
__device__ __forceinline__ void key_range(const EStore &S, u64 key, u64 *lo, u64 *hi) {
    *lo = *hi = 0;
    if (!S.nkey) return;
    const u64 a = lb64(S.key, 0, S.nkey, key);
    if (a < S.nkey && S.key[a] == key) { *lo = S.ptr[a]; *hi = S.ptr[a + 1]; }
}
// the key's ids in (me \ me_dm) u me_dp, ascending, handed to f until it returns false; returns how many were handed
template <class F>
__device__ u64 merged_ids(const EType &t, u64 key, F f) {
    u64 a, ae, d, de, p, pe;
    key_range(t.me, key, &a, &ae);
    key_range(t.medm, key, &d, &de);
    key_range(t.medp, key, &p, &pe);
    u64 k = 0;
    while (true) {
        while (a < ae) {                                     // skip deleted base ids
            const u64 va = t.me.id[a];
            while (d < de && t.medm.id[d] < va) d++;
            if (d < de && t.medm.id[d] == va) a++; else break;
        }
        const bool ha = a < ae, hp = p < pe;
        if (!ha && !hp) break;
        const u64 va = ha ? t.me.id[a] : 0, vp = hp ? t.medp.id[p] : 0;
        u64 v;
        if (ha && (!hp || va <= vp)) { v = va; a++; if (hp && vp == va) p++; }
        else { v = vp; p++; }
        k++;
        if (!f(k - 1, v)) break;
    }
    return k;
}

// edges.cu: the adjacency of n >= 1 distinct nodes d_src (device) over T types dt (device), in Graph::get_node_relationships_by_type's
// order (graph.rs:1797-1835): per node, types in order; per type the outgoing half (neighbour ascending, ids ascending), then the
// incoming half (source ascending); under dir 2 a self-loop once, in the outgoing half.  Device outputs: node i covers
// p[i] .. p[i+1] of node (the neighbour) and edge (the id); with tb, per entry its type << 1 | 1 for the incoming half.  Returns
// the entries; adds the passes' compulsory bytes to *bytes.
u64 edge_adjacency(const ETypes &types, const u64 *d_src, u64 n, int dir, DevBuf<u64> &p, DevBuf<u32> &node, DevBuf<u64> &edge,
                   u64 *bytes, DevBuf<u32> *tb = nullptr);

// edges.cu: row[i] = the row of keys[i]'s node among the nu distinct nodes u (ascending); with adj_p also deg[i] = the row's
// adjacency length, and deg[n] = 0.  A key's node is its low word: a u32 node, or a (slot << 32 | v) key.
template <class K> void node_rows(const K *keys, u64 n, const u64 *u, u64 nu, const u64 *adj_p, u32 *row, u64 *deg);
// edges.cu: the adjacency (direction dir, with each entry's type and half when want_tb) of the distinct nodes u of keys[0 .. n),
// per key its row, and cum = the scan of the rows' lengths (cum[n] = total).  Adds edge_adjacency's compulsory bytes to *bytes;
// the rest of the fetch is in the caller's formula.
struct NodeAdj {
    DevBuf<u64> u, p, edge, cum;
    DevBuf<u32> node, tb, row;
    u64 total = 0;
    template <class K> void fetch(const ETypes &types, const K *keys, u64 n, int dir, bool want_tb, u64 *bytes);
};

// ---- batched pair searches (shortest_path.cu, all_shortest_paths.cu) ----
// Pairs run in slices of slots, and a slot's entries are keyed (slot << 32 | v).
static const u64 SLOT_NONE = ~0ULL;
static const int SLOT_KEY_BITS = 43;          // slot (< 1024) << 32 | v, and SLOT_NONE above every key in the low 43 bits
static const u32 PAIR_T = 256;

__device__ __forceinline__ bool slot_seen(const u64 *__restrict__ vis, u64 nw, u64 slot, u32 v) {
    return (vis[slot * nw + (v >> 6)] >> (v & 63)) & 1;
}
// neighbour entries per piece of a level: the caller's budget, or by default a sixteenth of the free memory at about 80 bytes
// per entry (keys, ranks, the sort's second buffers, run heads and their scans), below the sort's 2^31 keys
inline u64 piece_budget(u64 budget, size_t free_bytes) {
    return budget ? budget : std::min<u64>((u64)1 << 30, std::max<u64>((u64)1 << 16, free_bytes / 16 / 80));
}
// edges.cu: front entries [0, nf), whose neighbour entries cum scans (cum[nf] = total), cut into rank-ordered pieces of at most
// budget neighbour entries (a piece holds at least one front entry); f(i0, i1, q0, q1) per piece that has entries: front
// entries [i0, i1), neighbour entries [q0, q1)
void for_each_piece(const u64 *cum, u64 nf, u64 total, u64 budget, const std::function<void(u64, u64, u64, u64)> &f);
// edges.cu: run_slice(p0, S) over the np pairs in slices of at most S_max.  A slice that runs out of device memory is run again
// as two halves (down to one pair), so a large batch on a large graph slices instead of failing.  A rerun slice must start from
// the state its failed run found, so run_slice commits its results only once nothing can fail.
void for_each_slice(u64 np, u64 S_max, const std::function<void(u64, u64)> &run_slice);

// capacity for need entries in b, keeping the first used
template <class T>
void grow(DevBuf<T> &b, u64 used, u64 need) {
    if (b.n >= need) return;
    DevBuf<T> nb(std::max<u64>(need, 2 * b.n));
    d2d(nb.ptr, b.ptr, used);
    b = std::move(nb);
}

} // namespace b200
