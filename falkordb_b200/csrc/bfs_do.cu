// bfs_do.cu -- direction-optimising BFS, one engine for a single GPU and for the 1-D row-block partition (BASELINE config 5,
// SURVEY 8e): level / min-id parent vectors as the reference consumes LAGr_BreadthFirstSearch_Extended
// (graph/src/runtime/functions/algo_procedures.rs:1079-1148, lagraphx_bindings.rs:585-594: max_level cap, dest early exit).
//
// Rank g owns vertices [lo, hi): their out-edges (row block of A) and their in-edges (row block of A').  Replicated on every
// rank, n bits each: `visited`, `frontier` (the previous level) and `newb` (the level being discovered); plus the global
// out-degree table (u32[n]).  Every rank therefore takes the same control decisions with no extra collective.
//   top-down level : expand the owned part of the frontier (flat, load-balanced) into a "discovered" set, exchange it,
//                    merge (drop visited); owned new vertices then find their parent = the first frontier member in their row
//                    of A' (rows ascend, so the first hit is the minimum id -- the oracle's tie-break)
//   bottom-up level: every owned unvisited vertex scans its row of A' for a frontier member and stops at the first hit
//                    (level and min-id parent in one step); only the owned slices of `newb` are exchanged
// Exchange over NCCL on the library stream: top-down ships the n-bit discovered bitmap of every rank (all-gather, OR-merge) or,
// when the frontier's out-edges number fewer than n/32 (density < 1/32, SURVEY 8e), sentinel-padded u32 lists of the discovered
// vertices; bottom-up all-gathers the owned n/P-bit slices in place.  Switch rule (Beamer): bottom-up while the frontier's
// out-edges exceed 1/ALPHA of the unexplored edges, back to top-down when the frontier shrinks below n/BETA.
// One small host read per level (frontier size / edges / dest flag) steers the loop; nothing else leaves the device.
//
// Without A' (one BFS on a fresh matrix, where building the mirror would cost more than the search) bfs_run runs a plain
// top-down BFS on one GPU with the same level and min-id parent; it has no dest early exit.
//
// Over relationship operands with pending writes (one GPU) the same loop walks A = U_t (m_t \ dm_t) u dp_t without building it:
// the kernels read a small array of operands {m, m', dp, dp', dm, dm'} (the DIRTY instantiations; DIRTY = false is the clean
// engine above).  Top-down expands one list per (frontier vertex, operand, layer m / dp) and skips an m entry found in the
// vertex's dm row; the parent and the bottom-up step take the minimum over the operands of the first frontier member in
// m'(v,:) \ dm'(v,:) and in dp'(v,:).  The switch reads sum_t deg(m_t) + deg(dp_t), an upper bound of the effective out-degree:
// it steers the direction only, levels and parents do not depend on it.
#include "common.cuh"
#include "ops.cuh"
#include <nccl.h>
#include <dlfcn.h>
#include <cstring>

namespace b200 {

static const u64 DO_CHUNK = 8192;
static const u64 DO_ALPHA = 14, DO_BETA = 24;

// ---------------------------------------------------------------------------------------------- NCCL, resolved at run time
// libb200grb.so carries no link-time dependency on NCCL: the reference links this library in place of GraphBLAS and only a
// multi-GPU deployment needs the collective.  In a torch process the already-loaded libnccl.so.2 is reused.
struct NcclApi {
    void *h = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    const char *(*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};
static NcclApi &nccl() {
    static NcclApi a;
    if (a.h || a.ok) return a;
    for (const char *name : {"libnccl.so.2", "libnccl.so"}) { a.h = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (a.h) break; }
    if (!a.h) return a;
    a.GetUniqueId = (decltype(a.GetUniqueId))dlsym(a.h, "ncclGetUniqueId");
    a.CommInitRank = (decltype(a.CommInitRank))dlsym(a.h, "ncclCommInitRank");
    a.CommDestroy = (decltype(a.CommDestroy))dlsym(a.h, "ncclCommDestroy");
    a.AllGather = (decltype(a.AllGather))dlsym(a.h, "ncclAllGather");
    a.GetErrorString = (decltype(a.GetErrorString))dlsym(a.h, "ncclGetErrorString");
    a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather;
    return a;
}
#define NCCL_TRY(expr)                                                                                          \
    do {                                                                                                        \
        ncclResult_t r__ = (expr);                                                                              \
        if (r__ != ncclSuccess)                                                                                 \
            throw GrbError(-7002, std::string("NCCL: ") + (nccl().GetErrorString ? nccl().GetErrorString(r__) : "error")); \
    } while (0)

struct BfsComm { ncclComm_t comm = nullptr; int rank = 0, world = 1; };

void comm_unique_id(unsigned char *id128) {
    if (!nccl().ok) throw GrbError(-7002, "NCCL (libnccl.so.2) is not available in this process");
    ncclUniqueId id;
    NCCL_TRY(nccl().GetUniqueId(&id));
    static_assert(sizeof(id) == 128, "ncclUniqueId is 128 bytes");
    memcpy(id128, &id, 128);
}
BfsComm *comm_init(int rank, int world, const unsigned char *id128) {
    if (world < 1 || rank < 0 || rank >= world) throw GrbError(-3, "comm_init: bad rank / world");
    BfsComm *c = new BfsComm();
    c->rank = rank; c->world = world;
    if (world > 1) {
        if (!nccl().ok) { delete c; throw GrbError(-7002, "NCCL (libnccl.so.2) is not available in this process"); }
        ncclUniqueId id;
        memcpy(&id, id128, 128);
        ensure_init();
        ncclResult_t r = nccl().CommInitRank(&c->comm, world, id, rank);
        if (r != ncclSuccess) { delete c; throw GrbError(-7002, "ncclCommInitRank failed"); }
    }
    return c;
}
void comm_free(BfsComm *c) {
    if (!c) return;
    if (c->comm) nccl().CommDestroy(c->comm);
    delete c;
}
int comm_rank(const BfsComm *c) { return c ? c->rank : 0; }
int comm_world(const BfsComm *c) { return c ? c->world : 1; }
void comm_allgather(BfsComm *c, const void *send, void *recv, size_t bytes_per_rank) {   // on the library stream
    if (!c || c->world == 1) { if (send != recv) CUDA_TRY(cudaMemcpyAsync(recv, send, bytes_per_rank, cudaMemcpyDeviceToDevice, stream())); return; }
    NCCL_TRY(nccl().AllGather(send, recv, bytes_per_rank, ncclUint8, c->comm, stream()));
}

// ---------------------------------------------------------------------------------------------- kernels
__device__ __forceinline__ bool bit_of(const u64 *__restrict__ b, u64 v) { return (b[v >> 6] >> (v & 63)) & 1ULL; }

// one operand of the dirty BFS on the device: the base m and its transpose mirror, dp and dm and their transposes (p null: empty)
struct BfsOpDev {
    const u64 *mp, *mtp, *dpp, *dptp, *dmp, *dmtp;
    const u32 *mj, *mtj, *dpj, *dptj, *dmj, *dmtj;
};

// the minimum-id frontier member of v's effective in-row, -1 if none, for one 8-lane group (every lane gets it).  Per operand
// m'(v,:) minus dm'(v,:) -- both rows ascend, so each lane's lower bound in dm' only moves forward -- then dp'(v,:).  Rows
// ascend, so a list stops at its first hit or once its entries pass the best hit so far.
__device__ __forceinline__ i64 do_first_parent(const BfsOpDev *__restrict__ ops, u32 nops, u64 v, const u64 *__restrict__ frontier,
                                               u32 lane8, u32 gmask) {
    u64 best = ~0ULL;
    for (u32 t = 0; t < nops; t++) {
        for (int layer = 0; layer < 2; layer++) {
            const u64 *Tp = layer ? ops[t].dptp : ops[t].mtp;
            const u32 *Tj = layer ? ops[t].dptj : ops[t].mtj;
            if (!Tp) continue;
            const u64 s = Tp[v], e = Tp[v + 1];
            u64 d = 0, de = 0;
            const u32 *Dj = ops[t].dmtj;
            if (!layer && ops[t].dmtp) { d = ops[t].dmtp[v]; de = ops[t].dmtp[v + 1]; }
            for (u64 qb = s; qb < e && Tj[qb] < best; qb += 8) {
                const u64 q = qb + lane8;
                u32 u = 0;
                bool hit = false;
                if (q < e) {
                    u = Tj[q];
                    hit = u < best && bit_of(frontier, u);
                    if (hit && d < de) {       // lb32 here reorders the code of k_do_pull<true> / k_do_assign<true>
                        u64 lo = d, hi = de;
                        while (lo < hi) { const u64 mid = (lo + hi) >> 1; if (Dj[mid] < u) lo = mid + 1; else hi = mid; }
                        d = lo;
                        if (d < de && Dj[d] == u) hit = false;      // a deleted edge
                    }
                }
                const u32 m = __ballot_sync(gmask, hit) & gmask;
                if (m) { best = __shfl_sync(gmask, u, __ffs(m) - 1); break; }
            }
        }
    }
    return best == ~0ULL ? -1 : (i64)best;
}

__global__ void k_do_deg32(const u64 *__restrict__ p, u64 nloc, u32 *__restrict__ deg) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < nloc; t += stride) { u64 d = p[t + 1] - p[t]; deg[t] = d > 0xFFFFFFFFULL ? 0xFFFFFFFFu : (u32)d; }
}
// deg += base (a base's cached table) + the row lengths of p (may be null), saturating
__global__ void k_do_deg_add(const u32 *__restrict__ base, const u64 *__restrict__ p, u64 n, u32 *__restrict__ deg) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        const u64 d = (u64)deg[t] + base[t] + (p ? p[t + 1] - p[t] : 0);
        deg[t] = d > 0xFFFFFFFFULL ? 0xFFFFFFFFu : (u32)d;
    }
}
__global__ void k_do_init(i64 *__restrict__ level, i64 *__restrict__ parent, u64 nloc, u64 lo, u64 src) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < nloc; t += stride) {
        const bool s = (t + lo == src);
        level[t] = s ? 0 : -1;
        if (parent) parent[t] = s ? (i64)src : -1;
    }
}
__global__ void k_do_set_bit(u64 *__restrict__ a, u64 *__restrict__ b, u64 v) { a[v >> 6] |= 1ULL << (v & 63); if (b) b[v >> 6] |= 1ULL << (v & 63); }

// set bits of words [w0, w1) of `bits` -> vertex list (any order), warp-aggregated
__global__ void __launch_bounds__(256) k_do_compact(const u64 *__restrict__ bits, u64 w0, u64 w1, u32 *__restrict__ list, u64 *__restrict__ count) {
    u64 w = w0 + (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u32 lane = threadIdx.x & 31;
    for (u64 base = w - lane; base < w1; base += stride) {
        const u64 ww = base + lane;
        u64 x = ww < w1 ? bits[ww] : 0ULL;
        u32 c = __popcll(x), incl = c;
#pragma unroll
        for (u32 d = 1; d < 32; d <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
        const u32 tot = __shfl_sync(0xffffffffu, incl, 31);
        if (!tot) continue;
        u64 at = 0;
        if (lane == 31) at = atomicAdd((unsigned long long *)count, (unsigned long long)tot);
        at = __shfl_sync(0xffffffffu, at, 31) + incl - c;
        while (x) { const u32 b = __ffsll((long long)x) - 1; x &= x - 1; list[at++] = (u32)((ww << 6) + b); }
    }
}
__global__ void k_do_frontier_deg(const u32 *__restrict__ fr, u64 nf, u64 lo, const u64 *__restrict__ Ap, u64 *__restrict__ deg, u64 *__restrict__ start) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t <= nf; t += stride) {
        if (t == nf) { deg[t] = 0; break; }
        const u64 u = fr[t] - lo;
        const u64 s = Ap[u];
        deg[t] = Ap[u + 1] - s;
        start[t] = s;
    }
}
// dirty top-down lists: list s = (frontier vertex s / nops2, operand (s % nops2) / 2, layer m / dp by s & 1)
__global__ void k_do_frontier_deg_delta(const u32 *__restrict__ fr, u64 nseg, const BfsOpDev *__restrict__ ops, u32 nops2,
                                        u64 *__restrict__ deg, u64 *__restrict__ start) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t <= nseg; t += stride) {
        if (t == nseg) { deg[t] = 0; break; }
        const u32 r = (u32)(t % nops2);
        const u64 *p = (r & 1) ? ops[r >> 1].dpp : ops[r >> 1].mp;
        const u64 u = fr[t / nops2];
        const u64 s = p ? p[u] : 0;
        deg[t] = p ? p[u + 1] - s : 0;
        start[t] = s;
    }
}
// top-down: every out-edge of the owned frontier vertices marks its unvisited target in `disc`.  DIRTY: the lists of
// k_do_frontier_deg_delta over the frontier `fr`; an m entry (u, v) in dm's row u is skipped (only a non-empty row searches).
template <bool DIRTY>
__global__ void __launch_bounds__(256)
k_do_expand(const u64 *__restrict__ cum, const u64 *__restrict__ start, u64 nf, u64 total, const u32 *__restrict__ Aj,
            const u64 *__restrict__ visited, u32 *__restrict__ disc, const u32 *__restrict__ fr, const BfsOpDev *__restrict__ ops,
            u32 nops2) {
    for (u64 chunk = blockIdx.x; chunk * DO_CHUNK < total; chunk += gridDim.x) {
        u64 lo = chunk * DO_CHUNK, hi = lo + DO_CHUNK;
        if (hi > total) hi = total;
        __syncthreads();
        for_each_flop(cum, 0, nf, lo, hi, [&](u64 e, u64 t) {
            if constexpr (DIRTY) {
                const u32 r = (u32)(e % nops2);
                const BfsOpDev &o = ops[r >> 1];
                const u32 v = ((r & 1) ? o.dpj : o.mj)[start[e] + (t - cum[e])];
                if (bit_of(visited, v)) return;
                if (!(r & 1) && o.dmp) {
                    const u64 u = fr[e / nops2];
                    const u64 s = o.dmp[u], de = o.dmp[u + 1];
                    if (s < de) {
                        const u64 d = lb32(o.dmj, s, de, v);
                        if (d < de && o.dmj[d] == v) return;   // a deleted edge
                    }
                }
                atomicOr(&disc[v >> 5], 1u << (v & 31));
            } else {
                const u32 v = Aj[start[e] + (t - cum[e])];
                if (!bit_of(visited, v)) atomicOr(&disc[v >> 5], 1u << (v & 31));
            }
        });
    }
}
// new = (OR of the P gathered bitmaps) & ~visited
__global__ void k_do_merge_or(const u64 *__restrict__ gathered, int P, u64 nw, const u64 *__restrict__ visited, u64 *__restrict__ newb) {
    u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; w < nw; w += stride) {
        u64 d = 0;
        for (int g = 0; g < P; g++) d |= gathered[(u64)g * nw + w];
        newb[w] = d & ~visited[w];
    }
}
// sparse exchange: sentinel-padded vertex lists of all ranks -> bits of newb (unvisited only; newb zeroed before)
__global__ void k_do_scatter_lists(const u32 *__restrict__ lists, u64 total, const u64 *__restrict__ visited, u32 *__restrict__ newb32) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < total; t += stride) {
        const u32 v = lists[t];
        if (v != 0xFFFFFFFFu && !bit_of(visited, v)) atomicOr(&newb32[v >> 5], 1u << (v & 31));
    }
}
// top-down epilogue: each owned new vertex takes the level and its minimum-id parent = first frontier member of its A' row
// (DIRTY: do_first_parent over the operands)
template <bool DIRTY>
__global__ void __launch_bounds__(256)
k_do_assign(const u32 *__restrict__ list, u64 cnt, u64 lo, const u64 *__restrict__ ATp, const u32 *__restrict__ ATj,
            const u64 *__restrict__ frontier, i64 *__restrict__ level, i64 *__restrict__ parent, i64 lvl,
            const BfsOpDev *__restrict__ ops, u32 nops) {
    const u32 lane8 = threadIdx.x & 7, sub = (threadIdx.x & 31) >> 3;
    const u32 gmask = 0xFFu << (8 * sub);
    u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 ng = ((u64)gridDim.x * blockDim.x) >> 3;
    for (u64 base = g - sub; base < cnt; base += ng) {
        const u64 i = base + sub;
        if (i >= cnt) continue;                      // uniform inside the 8-lane group
        const u64 r = list[i] - lo;
        i64 par = -1;
        if constexpr (DIRTY) {
            if (parent) par = do_first_parent(ops, nops, r + lo, frontier, lane8, gmask);
        } else if (parent) {
            const u64 s = ATp[r], e = ATp[r + 1];
            for (u64 qb = s; qb < e; qb += 8) {
                const u64 q = qb + lane8;
                u32 u = 0;
                bool hit = false;
                if (q < e) { u = ATj[q]; hit = bit_of(frontier, u); }
                const u32 m = __ballot_sync(gmask, hit) & gmask;
                if (m) { par = (i64)__shfl_sync(gmask, u, __ffs(m) - 1); break; }
            }
        }
        if (lane8 == 0) { level[r] = lvl; if (parent) parent[r] = par; }
    }
}
// bottom-up: owned unvisited vertices look for a frontier in-neighbour; first hit in ascending order = minimum-id parent
// (DIRTY: do_first_parent over the operands)
template <bool DIRTY>
__global__ void __launch_bounds__(256)
k_do_pull(const u64 *__restrict__ ATp, const u32 *__restrict__ ATj, u64 nloc, u64 lo, const u64 *__restrict__ frontier,
          const u64 *__restrict__ visited, u32 *__restrict__ newb32, i64 *__restrict__ level, i64 *__restrict__ parent, i64 lvl,
          const BfsOpDev *__restrict__ ops, u32 nops) {
    const u32 lane8 = threadIdx.x & 7, sub = (threadIdx.x & 31) >> 3;
    const u32 gmask = 0xFFu << (8 * sub);
    u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 ng = ((u64)gridDim.x * blockDim.x) >> 3;
    for (u64 base = g - sub; base < nloc; base += ng) {
        const u64 r = base + sub;
        if (r >= nloc) continue;
        const u64 v = lo + r;
        if (bit_of(visited, v)) continue;
        if constexpr (DIRTY) {
            const i64 par = do_first_parent(ops, nops, v, frontier, lane8, gmask);
            if (par >= 0 && lane8 == 0) {
                atomicOr(&newb32[v >> 5], 1u << (v & 31));
                level[r] = lvl;
                if (parent) parent[r] = par;
            }
            continue;
        }
        const u64 s = ATp[r], e = ATp[r + 1];
        for (u64 qb = s; qb < e; qb += 8) {
            const u64 q = qb + lane8;
            u32 u = 0;
            bool hit = false;
            if (q < e) { u = ATj[q]; hit = bit_of(frontier, u); }
            const u32 m = __ballot_sync(gmask, hit) & gmask;
            if (m) {
                const u32 par = __shfl_sync(gmask, u, __ffs(m) - 1);
                if (lane8 == 0) {
                    atomicOr(&newb32[v >> 5], 1u << (v & 31));
                    level[r] = lvl;
                    if (parent) parent[r] = (i64)par;
                }
                break;
            }
        }
    }
}
// visited |= new; st[0] = |new|, st[1] = out-edges of new, st[2] = dest reached
__global__ void __launch_bounds__(256)
k_do_stats(const u64 *__restrict__ newb, u64 nw, u64 *__restrict__ visited, const u32 *__restrict__ deg_all, u64 dest, u64 *__restrict__ st) {
    u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 cnt = 0, ed = 0;
    for (; w < nw; w += stride) {
        u64 x = newb[w];
        if (!x) continue;
        visited[w] |= x;
        cnt += __popcll(x);
        if (dest != ~0ULL && (dest >> 6) == w && ((x >> (dest & 63)) & 1ULL)) st[2] = 1;
        while (x) { const u32 b = __ffsll((long long)x) - 1; x &= x - 1; ed += deg_all[(w << 6) + b]; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) { cnt += __shfl_xor_sync(0xffffffffu, cnt, o); ed += __shfl_xor_sync(0xffffffffu, ed, o); }
    if ((threadIdx.x & 31) == 0 && cnt) { atomicAdd((unsigned long long *)&st[0], cnt); atomicAdd((unsigned long long *)&st[1], ed); }
}

// ---------------------------------------------------------------------------------------------- top-down only (no A')
__global__ void k_bfs_init(i64 *__restrict__ level, i64 *__restrict__ parent, u64 *__restrict__ cand, u64 n, u64 src) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n; t += stride) {
        level[t] = (t == src) ? 0 : -1;
        if (parent) parent[t] = (t == src) ? (i64)src : -1;
        cand[t] = ~0ULL;
    }
}

// PHASE 0: cand[v] = min(cand[v], u) for unvisited v.  PHASE 1: the winning (u,v) claims v.
template <int PHASE>
__global__ void __launch_bounds__(256)
k_bfs_expand(const u32 *__restrict__ fr, const u64 *__restrict__ cum, const u64 *__restrict__ start, u64 nf, u64 total,
             const u32 *__restrict__ Aj, i64 *__restrict__ level, i64 *__restrict__ parent, u64 *__restrict__ cand,
             i64 next_level, u32 *__restrict__ next, u32 *__restrict__ next_count) {
    u64 lo = (u64)blockIdx.x * DO_CHUNK, hi = lo + DO_CHUNK;
    if (hi > total) hi = total;
    for_each_flop(cum, 0, nf, lo, hi, [&](u64 e, u64 t) {
        u32 u = fr[e];
        u32 v = Aj[start[e] + (t - cum[e])];
        if (PHASE == 0) {
            if (level[v] < 0) atomicMin((unsigned long long *)&cand[v], (unsigned long long)u);
        } else {
            // level[v] is only ever written here, by the unique (u,v) with u == cand[v]
            if (cand[v] == (u64)u && level[v] < 0) {
                level[v] = next_level;
                if (parent) parent[v] = (i64)u;
                next[atomicAdd(next_count, 1u)] = v;
            }
        }
    });
}

// ---------------------------------------------------------------------------------------------- driver
// deg_all: device u32[n_pad] (out-degrees of every vertex, replicated); total_edges = sum of it.
void bfs_build_degrees(const DevCSR &Aloc, u64 n, u64 lo, u64 hi, BfsComm *comm, DevBuf<u32> &deg_all, u64 *total_edges) {
    const int P = comm_world(comm);
    const u64 block = P > 1 ? (n + P - 1) / P : n;
    if (P > 1 && (block % 64 || lo != (u64)comm_rank(comm) * block)) throw GrbError(-3, "partitioned BFS: row blocks must be ceil(n / P) rounded to 64 vertices");
    deg_all.alloc(block * P);
    deg_all.zero();
    const u64 nloc = hi - lo;
    if (nloc) LAUNCH(k_do_deg32, grid_for(nloc, 256, (u64)ctx().num_sms * 16), 256, 0, Aloc.p.ptr, nloc, deg_all.ptr + lo);
    if (P > 1) comm_allgather(comm, deg_all.ptr + lo, deg_all.ptr, block * sizeof(u32));
    DevBuf<u64> nnz(1);
    CUDA_TRY(cudaMemcpyAsync(nnz.ptr, Aloc.p.ptr + nloc, sizeof(u64), cudaMemcpyDeviceToDevice, stream()));
    u64 local = read_scalar(nnz.ptr);
    if (P > 1) {        // total over ranks: gather the P local counts
        DevBuf<u64> all(P);
        CUDA_TRY(cudaMemcpyAsync(all.ptr + comm_rank(comm), nnz.ptr, sizeof(u64), cudaMemcpyDeviceToDevice, stream()));
        comm_allgather(comm, all.ptr + comm_rank(comm), all.ptr, sizeof(u64));
        std::vector<u64> h(P);
        CUDA_TRY(cudaMemcpyAsync(h.data(), all.ptr, P * sizeof(u64), cudaMemcpyDeviceToHost, stream()));
        sync_stream();
        local = 0;
        for (u64 x : h) local += x;
    }
    *total_edges = local;
}

// the switch's table over dirty operands, per call: sum_t deg(m_t) (each base's cached table) + deg(dp_t)
void bfs_delta_degrees(const std::vector<BfsOperand> &ops, u64 n, DevBuf<u32> &deg, u64 *total_edges) {
    deg.alloc(n ? n : 1);
    deg.zero();
    u64 total = 0;
    for (const BfsOperand &o : ops) {
        if (n) LAUNCH(k_do_deg_add, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, o.deg, o.dp ? o.dp->p.ptr : (const u64 *)nullptr, n, deg.ptr);
        total += o.edges + (o.dp ? o.dp->nnz : 0);
    }
    *total_edges = total;
}

static const u64 *csr_p(const DevCSR *A) { return A ? A->p.ptr : nullptr; }
static const u32 *csr_j(const DevCSR *A) { return A ? A->j.ptr : nullptr; }

void bfs_do(const DevCSR &Aloc, const DevCSR &ATloc, u64 n, u64 lo, u64 hi, const u32 *deg_all, u64 total_edges, BfsComm *comm,
            u64 src, i64 max_level, i64 dest, i64 *d_level, i64 *d_parent, BfsInfo *info, const std::vector<BfsOperand> *dirty) {
    if (src >= n) throw GrbError(-4, "BFS source out of range");
    const int P = comm_world(comm), rank = comm_rank(comm);
    if (dirty && (P > 1 || dirty->empty())) throw GrbError(-3, "BFS over operands with deltas: one GPU and at least one operand");
    // the dirty operands on the device; layers: transposed rows a parent search reads per vertex (for the byte counts)
    const u32 nops = dirty ? (u32)dirty->size() : 0;
    DevBuf<BfsOpDev> dops;
    std::vector<BfsOpDev> h(nops);
    u64 layers = 0;
    if (dirty) {
        for (u32 t = 0; t < nops; t++) {
            const BfsOperand &o = (*dirty)[t];
            h[t] = BfsOpDev{csr_p(o.m), csr_p(o.mT), csr_p(o.dp), csr_p(o.dpT), csr_p(o.dm), csr_p(o.dmT),
                            csr_j(o.m), csr_j(o.mT), csr_j(o.dp), csr_j(o.dpT), csr_j(o.dm), csr_j(o.dmT)};
            layers += 1 + (o.dpT != nullptr) + (o.dmT != nullptr);
        }
        dops.alloc(nops);
        h2d(dops.ptr, h.data(), nops);
    }
    const u64 block = P > 1 ? (n + P - 1) / P : n;          // vertices per rank (multiple of 64 when P > 1)
    const u64 nwl = P > 1 ? block / 64 : (n + 63) / 64;     // words per owned slice
    const u64 nw = nwl * P;                                 // words of a replicated bitmap (padded)
    const u64 nloc = hi - lo;
    Context &cx = ctx();
    DevBuf<u64> visited(nw), fa(nw), fb(nw), disc(nw), st(4);
    DevBuf<u64> gather;
    visited.zero(); fa.zero();
    u64 *frontier = fa.ptr, *newb = fb.ptr;
    if (nloc) LAUNCH(k_do_init, grid_for(nloc, 256, (u64)ctx().num_sms * 16), 256, 0, d_level, d_parent, nloc, lo, src);
    LAUNCH(k_do_set_bit, 1, 1, 0, visited.ptr, frontier, src);
    u32 dsrc = 0;
    d2h(&dsrc, deg_all + src, 1);
    sync_stream();
    u64 nf = 1, mf = dsrc, explored = dsrc, edges = dsrc, reached = 1;
    const u64 udest = dest >= 0 ? (u64)dest : ~0ULL;
    bool bottom_up = false;
    i64 lvl = 0;
    BfsInfo rec;
    memset(&rec, 0, sizeof(rec));
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    if (info) { CUDA_TRY(cudaEventCreate(&ev0)); CUDA_TRY(cudaEventCreate(&ev1)); }
    struct EvGuard { cudaEvent_t &a, &b; ~EvGuard() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); } } evg{ev0, ev1};
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> exch;   // per-level exchange brackets (timed after the run)
    auto exchange_begin = [&]() { if (info && P > 1) { cudaEvent_t a, b; CUDA_TRY(cudaEventCreate(&a)); CUDA_TRY(cudaEventCreate(&b)); CUDA_TRY(cudaEventRecord(a, stream())); exch.push_back({a, b}); } };
    auto exchange_end = [&]() { if (info && P > 1) CUDA_TRY(cudaEventRecord(exch.back().second, stream())); };
    if (info) CUDA_TRY(cudaEventRecord(ev0, stream()));
    while (nf > 0 && (max_level < 0 || lvl < max_level) && !(udest != ~0ULL && udest == src)) {
        const u64 unexplored = total_edges > explored ? total_edges - explored : 0;
        if (!bottom_up) { if (mf > unexplored / DO_ALPHA && cx.opt_bfs_direction != 1) bottom_up = true; }
        else if (nf < n / DO_BETA && cx.opt_bfs_direction != 2) bottom_up = false;
        if (cx.opt_bfs_direction == 1) bottom_up = false;
        if (cx.opt_bfs_direction == 2) bottom_up = true;
        lvl++;
        st.zero();
        if (!bottom_up) {
            // ---- top-down ----
            DevBuf<u32> list(nloc ? nloc : 1);
            DevBuf<u64> cnt(1);
            cnt.zero();
            const u64 w0 = (u64)rank * nwl * (P > 1), w1 = P > 1 ? w0 + nwl : nw;
            LAUNCH(k_do_compact, grid_for(w1 - w0, 256, (u64)ctx().num_sms * 8), 256, 0, frontier, w0, w1, list.ptr, cnt.ptr);
            const u64 nfl = read_scalar(cnt.ptr);
            disc.zero();
            if (nfl && dirty) {
                // one list per (frontier vertex, operand, layer m / dp)
                const u64 nseg = nfl * 2 * nops;
                DevBuf<u64> cum(nseg + 1), start(nseg);
                LAUNCH(k_do_frontier_deg_delta, grid_for(nseg + 1, 256, (u64)ctx().num_sms * 16), 256, 0, list.ptr, nseg, dops.ptr, 2 * nops, cum.ptr, start.ptr);
                exclusive_scan_u64(cum.ptr, cum.ptr, nseg + 1);
                const u64 total = read_scalar(cum.ptr + nseg);
                if (total) {
                    // column ids of every listed entry, each list's offset and start, each (vertex, operand)'s dm row pointers
                    TimedScope ts(TK_BFS_DELTA, 4 * total + 16 * nseg + 16 * nfl * nops);
                    const u32 grid = (u32)std::min<u64>((total + DO_CHUNK - 1) / DO_CHUNK, (u64)cx.num_sms * 16);
                    LAUNCH(k_do_expand<true>, grid, 256, 0, cum.ptr, start.ptr, nseg, total, (const u32 *)nullptr, visited.ptr, (u32 *)disc.ptr,
                           list.ptr, dops.ptr, 2 * nops);
                }
            } else if (nfl) {
                DevBuf<u64> cum(nfl + 1), start(nfl);
                LAUNCH(k_do_frontier_deg, grid_for(nfl + 1, 256, (u64)ctx().num_sms * 16), 256, 0, list.ptr, nfl, lo, Aloc.p.ptr, cum.ptr, start.ptr);
                exclusive_scan_u64(cum.ptr, cum.ptr, nfl + 1);
                const u64 total = read_scalar(cum.ptr + nfl);
                if (total) {
                    TimedScope ts(TK_BFS_EXPAND, 4 * total + 20 * nfl);
                    const u32 grid = (u32)std::min<u64>((total + DO_CHUNK - 1) / DO_CHUNK, (u64)cx.num_sms * 16);
                    LAUNCH(k_do_expand<false>, grid, 256, 0, cum.ptr, start.ptr, nfl, total, Aloc.j.ptr, visited.ptr, (u32 *)disc.ptr,
                           (const u32 *)nullptr, (const BfsOpDev *)nullptr, 0u);
                }
            }
            if (P == 1) {
                LAUNCH(k_do_merge_or, grid_for(nw, 256, (u64)ctx().num_sms * 8), 256, 0, disc.ptr, 1, nw, visited.ptr, newb);
            } else if (mf < n / 32 && cx.opt_bfs_sparse_exchange) {
                // sparse: a rank discovers at most mf vertices (the frontier's out-edges, known identically everywhere)
                const u64 bound = mf ? mf : 1;
                DevBuf<u32> mine(bound), all(bound * P);
                CUDA_TRY(cudaMemsetAsync(mine.ptr, 0xFF, bound * sizeof(u32), stream()));
                cnt.zero();
                LAUNCH(k_do_compact, grid_for(nw, 256, (u64)ctx().num_sms * 8), 256, 0, disc.ptr, (u64)0, nw, mine.ptr, cnt.ptr);
                exchange_begin();
                comm_allgather(comm, mine.ptr, all.ptr, bound * sizeof(u32));
                exchange_end();
                CUDA_TRY(cudaMemsetAsync(newb, 0, nw * sizeof(u64), stream()));
                LAUNCH(k_do_scatter_lists, grid_for(bound * P, 256, (u64)ctx().num_sms * 8), 256, 0, all.ptr, bound * P, visited.ptr, (u32 *)newb);
                rec.sparse_levels++;
                rec.exchanged_bytes += bound * sizeof(u32) * P;
            } else {
                if (!gather.ptr) gather.alloc(nw * P);
                exchange_begin();
                comm_allgather(comm, disc.ptr, gather.ptr, nw * sizeof(u64));
                exchange_end();
                LAUNCH(k_do_merge_or, grid_for(nw, 256, (u64)ctx().num_sms * 8), 256, 0, gather.ptr, P, nw, visited.ptr, newb);
                rec.exchanged_bytes += nw * sizeof(u64) * P;
            }
            // owned new vertices: level + min-id parent
            cnt.zero();
            LAUNCH(k_do_compact, grid_for(w1 - w0, 256, (u64)ctx().num_sms * 8), 256, 0, newb, w0, w1, list.ptr, cnt.ptr);
            const u64 nnew = read_scalar(cnt.ptr);
            if (nnew && dirty) {
                // the new vertices' list entries, levels and parents, and the transposed rows' pointers they read
                TimedScope ts(TK_BFS_DELTA, 20 * nnew + 16 * nnew * layers);
                LAUNCH(k_do_assign<true>, grid_for(nnew * 8, 256, (u64)ctx().num_sms * 16), 256, 0, list.ptr, nnew, lo, (const u64 *)nullptr,
                       (const u32 *)nullptr, frontier, d_level, d_parent, lvl, dops.ptr, nops);
            } else if (nnew) {
                LAUNCH(k_do_assign<false>, grid_for(nnew * 8, 256, (u64)ctx().num_sms * 16), 256, 0, list.ptr, nnew, lo, ATloc.p.ptr, ATloc.j.ptr,
                       frontier, d_level, d_parent, lvl, (const BfsOpDev *)nullptr, 0u);
            }
            rec.td_levels++;
        } else {
            // ---- bottom-up ----
            CUDA_TRY(cudaMemsetAsync(newb, 0, nw * sizeof(u64), stream()));
            if (nloc && dirty) {
                // the visited bitmap, and the transposed rows' pointers of every unvisited vertex
                TimedScope ts(TK_BFS_DELTA, 8 * nw + 16 * (n - reached) * layers);
                LAUNCH(k_do_pull<true>, grid_for(nloc * 8, 256, (u64)cx.num_sms * 32), 256, 0, (const u64 *)nullptr, (const u32 *)nullptr, nloc, lo,
                       frontier, visited.ptr, (u32 *)newb, d_level, d_parent, lvl, dops.ptr, nops);
            } else if (nloc) {
                TimedScope ts(TK_BFS_EXPAND, 0);
                LAUNCH(k_do_pull<false>, grid_for(nloc * 8, 256, (u64)cx.num_sms * 32), 256, 0, ATloc.p.ptr, ATloc.j.ptr, nloc, lo, frontier, visited.ptr,
                       (u32 *)newb, d_level, d_parent, lvl, (const BfsOpDev *)nullptr, 0u);
            }
            if (P > 1) {
                exchange_begin();
                comm_allgather(comm, newb + (u64)rank * nwl, newb, nwl * sizeof(u64));     // in place
                exchange_end();
                rec.exchanged_bytes += nw * sizeof(u64);
            }
            rec.bu_levels++;
        }
        LAUNCH(k_do_stats, grid_for(nw, 256, (u64)ctx().num_sms * 8), 256, 0, newb, nw, visited.ptr, deg_all, udest, st.ptr);
        u64 hst[3] = {0, 0, 0};
        d2h(hst, st.ptr, 3);
        sync_stream();
        nf = hst[0]; mf = hst[1];
        reached += nf;
        explored += mf; edges += mf;
        if (nf == 0) { lvl--; break; }
        u64 *t = frontier; frontier = newb; newb = t;
        if (hst[2]) break;                           // dest reached (lagraphx_bindings.rs:585-594)
    }
    if (info) {
        CUDA_TRY(cudaEventRecord(ev1, stream()));
        CUDA_TRY(cudaEventSynchronize(ev1));
        float ms = 0;
        cudaEventElapsedTime(&ms, ev0, ev1);
        rec.device_ms = ms;
        double ex = 0;
        for (auto &pr : exch) { float m = 0; if (cudaEventElapsedTime(&m, pr.first, pr.second) == cudaSuccess) ex += m; cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
        rec.exchange_ms = ex;
        rec.exchanges = (u64)exch.size();
        rec.depth = (u64)lvl;
        rec.edges = edges;
        *info = rec;
    }
}

// Top-down BFS over A alone.  The parent is made deterministic by a candidate pass before the claim pass: cand[v] = the minimum
// frontier id with an edge to v (atomicMin), so only that u claims v.
// Algorithmic bytes (SURVEY 8d): 4*m_visited*2 + 16*n_visited + 16*n_reached.
void bfs_run(const DevCSR &A, u64 src, i64 max_level, i64 *d_level, i64 *d_parent, u64 *edges_traversed) {
    u64 n = A.nrows;
    if (src >= n) throw GrbError(-4, "BFS source out of range");
    DevBuf<u64> cand(n);
    LAUNCH(k_bfs_init, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, d_level, d_parent, cand.ptr, n, src);
    DevBuf<u32> fa(n), fb(n), ncount(1);
    u32 s32 = (u32)src;
    h2d(fa.ptr, &s32, 1);
    u64 nf = 1, edges = 0;
    i64 lvl = 0;
    u32 *cur = fa.ptr, *nxt = fb.ptr;
    DevBuf<u64> cum(n + 1), start(n);
    while (nf > 0 && (max_level < 0 || lvl < max_level)) {
        LAUNCH(k_do_frontier_deg, grid_for(nf + 1, 256, (u64)ctx().num_sms * 16), 256, 0, cur, nf, (u64)0, A.p.ptr, cum.ptr, start.ptr);
        exclusive_scan_u64(cum.ptr, cum.ptr, nf + 1);
        u64 total = read_scalar(cum.ptr + nf);
        if (total == 0) break;
        edges += total;
        ncount.zero();
        u32 grid = (u32)((total + DO_CHUNK - 1) / DO_CHUNK);
        LAUNCH((k_bfs_expand<0>), grid, 256, 0, cur, cum.ptr, start.ptr, nf, total, A.j.ptr, d_level, d_parent, cand.ptr,
               lvl + 1, nxt, ncount.ptr);
        LAUNCH((k_bfs_expand<1>), grid, 256, 0, cur, cum.ptr, start.ptr, nf, total, A.j.ptr, d_level, d_parent, cand.ptr,
               lvl + 1, nxt, ncount.ptr);
        nf = read_scalar(ncount.ptr);
        u32 *t = cur; cur = nxt; nxt = t;
        lvl++;
    }
    if (edges_traversed) *edges_traversed = edges;
}

} // namespace b200
