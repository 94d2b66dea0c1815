// edge_layers.cuh -- a relationship Tensor's live layers as the device reads them, and the point lookups over them that both
// B200_expand_edges (edges.cu) and the write plans (writes.cu) make: find_rc, Tensor::eff_get, and a multi-edge pair's merged id
// list (me \ me_dm) u me_dp.
#pragma once
#include "common.cuh"
#include "ops.cuh"

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

__device__ __forceinline__ u64 lb32(const u32 *__restrict__ j, u64 lo, u64 hi, u32 c) {
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (j[mid] < c) lo = mid + 1; else hi = mid; }
    return lo;
}
__device__ __forceinline__ u64 ub32(const u32 *__restrict__ j, u64 lo, u64 hi, u32 c) {
    while (lo < hi) { u64 mid = (lo + hi) >> 1; if (j[mid] <= c) lo = mid + 1; else hi = mid; }
    return lo;
}
// largest g with lstart[g] <= e (lstart ascending, lstart[0] = 0): the segment of flat position e behind a scan of lengths
__device__ __forceinline__ u64 list_at(const u64 *__restrict__ lstart, u64 G, u64 e) {
    u64 lo = 0, hi = G - 1;
    while (lo < hi) { u64 mid = (lo + hi + 1) >> 1; if (lstart[mid] <= e) lo = mid; else hi = mid - 1; }
    return lo;
}
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
    u64 a = 0, b = S.nkey;
    while (a < b) { u64 mid = (a + b) >> 1; if (S.key[mid] < key) a = mid + 1; else b = mid; }
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
u64 edge_adjacency(const EType *dt, u32 T, const u64 *d_src, u64 n, int dir, DevBuf<u64> &p, DevBuf<u32> &node, DevBuf<u64> &edge,
                   u64 *bytes, DevBuf<u32> *tb = nullptr);

} // namespace b200
