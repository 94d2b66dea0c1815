// bits_hop.cu -- the bit-matrix hop Y = X * A: the push from the frontier's active vertices, the pull through A' with its segment
// list, hot-set tables and L2 policies, the choice between them (hop_impl), and the exact dirty-hop repair, which reuses the pull's
// lane split.
#include "frontier.cuh"

namespace b200 {

// flops (mxm sense) = sum_k popc(X[k]) * deg_A(k); edges = sum_{k active} deg_A(k); flag[k] = active
__global__ void __launch_bounds__(256)
k_bits_flops(const u64 *__restrict__ X, u32 W, u64 n, const u64 *__restrict__ Ap, u32 *__restrict__ flag,
             u64 *__restrict__ out /* [0]=flops [1]=edges */) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts, ts2;
    u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 fl = 0, ed = 0;
    for (; k < n; k += stride) {
        u32 pc = 0;
        for (u32 w = 0; w < W; w++) pc += __popcll(X[k * W + w]);
        u64 d = Ap[k + 1] - Ap[k];
        flag[k] = (pc != 0 && d != 0) ? 1u : 0u;
        if (pc) { fl += (u64)pc * d; ed += d; }
    }
    u64 tf = Red(ts).Sum(fl);
    u64 te = Red(ts2).Sum(ed);
    if (threadIdx.x == 0) {
        if (tf) atomicAdd((unsigned long long *)&out[0], tf);
        if (te) atomicAdd((unsigned long long *)&out[1], te);
    }
}

// ---------------------------------------------------------------------------- push
__global__ void k_compact_active(const u32 *__restrict__ flag, const u64 *__restrict__ pos, u64 n,
                                 const u64 *__restrict__ Ap, u32 *__restrict__ act, u64 *__restrict__ deg,
                                 u64 *__restrict__ astart) {
    u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; k < n; k += stride) {
        if (flag[k]) {
            u64 d = pos[k];
            act[d] = (u32)k;
            u64 s = Ap[k];
            deg[d] = Ap[k + 1] - s;
            astart[d] = s;
        }
    }
}

template <int W>
__global__ void __launch_bounds__(256)
k_bits_push(const u32 *__restrict__ act, const u64 *__restrict__ cum, const u64 *__restrict__ astart, u64 nact,
            u64 total, const u32 *__restrict__ Aj, const u64 *__restrict__ X, u64 *__restrict__ Y) {
    u64 lo = (u64)blockIdx.x * PUSH_CHUNK, hi = lo + PUSH_CHUNK;
    if (hi > total) hi = total;
    for_each_flop(cum, 0, nact, lo, hi, [&](u64 e, u64 t) {
        u32 k = act[e];
        u32 col = Aj[astart[e] + (t - cum[e])];
#pragma unroll
        for (int w = 0; w < W; w++) {
            u64 xw = X[(u64)k * W + w];
            if (xw) atomicOr((unsigned long long *)&Y[(u64)col * W + w], xw);
        }
    });
}

// ---------------------------------------------------------------------------- pull
// Y[j] = OR of X[k] over k in A'(j,:).  What bounds a pull is the L1TEX tag stage: one 128-byte line per clock per SM, and a
// warp-wide gather with every lane on a different vertex costs 32 of those "wavefronts" per instruction.  A vertex record of
// W = 8 words is 64 bytes -- one line -- but a lane can fetch at most 16 bytes per instruction on sm_90 (LDG.128), so
// one-lane-per-vertex spends FOUR wavefronts per vertex.  In k_pull_seg SPLIT = W / 2 adjacent lanes share a vertex: lane h loads
// words [2h, 2h+2) of the record with one LDG.128, the requests fall into the same line and coalesce into one wavefront, and the
// lanes never exchange data (each lane ORs, keeps and finally stores its own 16-byte part of the output row).
// W = 4 -> half the wavefronts per gathered vertex; W = 8 -> a quarter; W = 16 -> an eighth; W <= 2 keeps one lane per record.
// The rows of A' are binned once per matrix (build_pull_tables):
//   small (<= SMALL_ROW entries) : k_pull_small, one lane per row in natural order; it also zero-fills the long rows
//   mid   (<= LONG_ROW)          : k_pull_seg, 8 lanes per row, from a list sorted by length, descending
//   long                         : the same list, as LONG_ROW-entry segments whose partial results are merged with RED.OR
struct OrOp64 { __device__ u64 operator()(u64 a, u64 b) const { return a | b; } };

// G[w] = OR over all vertices of word w: the terminal value of the OR monoid for this frontier.  A pull row whose
// accumulator has reached G cannot change any more, so the rest of its neighbours need not be gathered (exact).
template <int W>
__global__ void __launch_bounds__(256) k_or_all(const u64 *__restrict__ X, u64 nv, u64 *__restrict__ G) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 acc[W];
#pragma unroll
    for (int w = 0; w < W; w++) acc[w] = 0;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < nv; t += stride) {
#pragma unroll
        for (int w = 0; w < W; w++) acc[w] |= X[t * W + w];
    }
#pragma unroll
    for (int w = 0; w < W; w++) {
        u64 r = Red(ts).Reduce(acc[w], OrOp64());
        __syncthreads();
        if (threadIdx.x == 0 && r) atomicOr((unsigned long long *)&G[w], r);
    }
}

// The L2 policies of one pull launch with hints on.  The gather source X (the packed frontier, hot-set order: out-degree
// descending) is evict_last over its first `hot` bytes and evict_first over the rest of its `tot` bytes, or evict_normal
// everywhere when hot = 0.  streams != 0: A' col_idx and rowptr, the segment list and the stores of Y are evict_first, so the
// 2 GB that pass through once do not push the hot records out.
struct PullHints {
    u32 hot = 0, tot = 0, streams = 0;
#ifdef __CUDACC__
    __device__ __forceinline__ u64 gather_policy(const void *X) const { return hot ? policy_range(X, hot, tot) : policy_normal(); }
    __device__ __forceinline__ u64 stream_policy() const { return streams ? policy_stream() : policy_normal(); }
#endif
};

// HINTS: every load of the pull kernels carries an L2 policy (PullHints).  A' col_idx and rowptr lines are shared by the loads of
// neighbouring lanes and unroll steps, so they keep their L1 allocation; only their L2 priority changes
template <bool HINTS> __device__ __forceinline__ u32 ld_col(const u32 *p, u64 strm) { return HINTS ? ld_nc_u32(p, strm) : __ldg(p); }
template <bool HINTS> __device__ __forceinline__ u64 ld_ptr(const u64 *p, u64 strm) { return HINTS ? ld_nc_u64(p, strm) : __ldg(p); }
template <bool HINTS> __device__ __forceinline__ u64 ld_x(const u64 *p, u64 keep) { return HINTS ? ld_nc_u64(p, keep) : __ldg(p); }
// acc |= the W frontier words of one vertex: ONE 16-byte load per word pair (a W=4 vertex is a single 32 B sector), so the
// number of L1TEX wavefronts per gathered vertex does not grow with W
template <int W, bool HINTS> __device__ __forceinline__ void or_words(u64 (&acc)[W], const u64 *__restrict__ p, u64 keep) {
    if (W == 1) { acc[0] |= ld_x<HINTS>(p, keep); return; }
    const ulonglong2 *q = reinterpret_cast<const ulonglong2 *>(p);
#pragma unroll
    for (int w2 = 0; w2 < W / 2; w2++) {
        ulonglong2 v = HINTS ? ld_nc_v2(q + w2, keep) : __ldg(q + w2);
        acc[2 * w2] |= v.x;
        acc[2 * w2 + 1] |= v.y;
    }
}

static const u32 SMALL_ROW = 8;
static const u64 LONG_ROW = 4096;   // pull: rows longer than this are split into LONG_ROW-entry segments

// HINTS: the store carries policy pol (Y is written once and read by the next pass, not by this kernel)
template <int W, bool HINTS = false> __device__ __forceinline__ void store_row(u64 *dst, const u64 (&acc)[W], u64 pol = 0) {
    if constexpr (W == 1) {
        if (HINTS) st_u64_stream(dst, acc[0], pol);
        else dst[0] = acc[0];
    } else {
#pragma unroll
        for (int w2 = 0; w2 < W / 2; w2++) {
            ulonglong2 *q = reinterpret_cast<ulonglong2 *>(dst) + w2;
            if (HINTS) st_v2_hint(q, make_ulonglong2(acc[2 * w2], acc[2 * w2 + 1]), pol);
            else *q = make_ulonglong2(acc[2 * w2], acc[2 * w2 + 1]);
        }
    }
}
template <int WL, bool HINTS = false> __device__ __forceinline__ void store_part(u64 *dst, const u64 (&acc)[WL], u64 pol = 0) {
    store_row<WL, HINTS>(dst, acc, pol);
}
// accumulate mode (union hops): dst |= acc, skipped when acc is empty.  Each record is owned by one lane (k_pull_small) or one
// 8-lane group (a mid row of k_pull_seg), so a plain read-modify-write is race-free
template <int WL> __device__ __forceinline__ void or_part(u64 *dst, u64 (&acc)[WL]) {
    u64 any = 0;
#pragma unroll
    for (int w = 0; w < WL; w++) any |= acc[w];
    if (!any) return;
    if constexpr (WL == 1) { dst[0] |= acc[0]; }
    else {
#pragma unroll
        for (int w2 = 0; w2 < WL / 2; w2++) {
            ulonglong2 v = reinterpret_cast<const ulonglong2 *>(dst)[w2];
            reinterpret_cast<ulonglong2 *>(dst)[w2] = make_ulonglong2(v.x | acc[2 * w2], v.y | acc[2 * w2 + 1]);
        }
    }
}

static const u32 SEG_ATOMIC = 0x80000000u;

// segments per row: 0 (small), 1 (mid), ceil(len / LONG_ROW) (long); maxlen = the longest row when it is longer than LONG_ROW
__global__ void k_seg_count(const u64 *__restrict__ p, u64 n, u32 *__restrict__ cnt, u64 *__restrict__ maxlen) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 mx = 0;
    for (; r <= n; r += stride) {
        if (r == n) { cnt[r] = 0; break; }
        u64 d = p[r + 1] - p[r];
        cnt[r] = d <= SMALL_ROW ? 0u : (u32)((d + LONG_ROW - 1) / LONG_ROW);
        if (d > mx) mx = d;
    }
    if (mx > LONG_ROW) atomicMax((unsigned long long *)maxlen, mx);
}
// key = LONG_ROW - seglen (ascending sort = longest first), value = position of the segment: row << 20 | index inside the row
__global__ void k_seg_emit(const u64 *__restrict__ p, u64 n, const u64 *__restrict__ pos, u64 *__restrict__ keys, u64 *__restrict__ vals) {
    u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; r < n; r += stride) {
        const u64 d = p[r + 1] - p[r];
        if (d <= SMALL_ROW) continue;
        u64 o = pos[r];
        for (u64 s = 0, i = 0; s < d; s += LONG_ROW, i++) {
            const u64 len = d - s < LONG_ROW ? d - s : LONG_ROW;
            keys[o] = LONG_ROW - len;
            vals[o] = (r << 20) | i;
            o++;
        }
    }
}
__global__ void k_seg_unpack(const u64 *__restrict__ vals, u64 ns, const u64 *__restrict__ p, u32 *__restrict__ s_row,
                             u32 *__restrict__ s_len, u64 *__restrict__ s_start) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ns) return;
    const u64 v = vals[i];
    const u32 r = (u32)(v >> 20);
    const u64 k = v & 0xFFFFFu;
    const u64 d = p[r + 1] - p[r];
    const u64 s = k * LONG_ROW;
    const u64 len = d - s < LONG_ROW ? d - s : LONG_ROW;
    s_row[i] = r;
    s_start[i] = p[r] + s;
    s_len[i] = (u32)len | (d > LONG_ROW ? SEG_ATOMIC : 0u);
}
static void build_seg_list(const DevCSR &AT, PullTables &pt) {
    const u64 n = AT.nrows;
    pt.ns = 0;
    pt.s_row.release(); pt.s_len.release(); pt.s_start.release();
    if (!n) return;
    DevBuf<u32> cnt(n + 1);
    DevBuf<u64> pos(n + 1), mx(1);
    mx.zero();
    LAUNCH(k_seg_count, grid_for(n + 1, 256, 1 << 16), 256, 0, AT.p.ptr, n, cnt.ptr, mx.ptr);
    // k_seg_emit addresses a segment as row << 20 | index inside the row
    if (read_scalar(mx.ptr) >= ((u64)LONG_ROW << 20)) throw GrbError(-8, "pull: a row of A' exceeds 2^32 entries");
    exclusive_scan_u32_to_u64(cnt.ptr, pos.ptr, n + 1);
    const u64 ns = read_scalar(pos.ptr + n);
    pt.ns = ns;
    if (!ns) return;
    DevBuf<u64> keys(ns), vals(ns);
    LAUNCH(k_seg_emit, grid_for(n, 256, 1 << 16), 256, 0, AT.p.ptr, n, pos.ptr, keys.ptr, vals.ptr);
    sort_pairs_u64(keys.ptr, vals.ptr, ns, 13);          // stable: rows ascending inside one length
    pt.s_row.alloc(ns); pt.s_len.alloc(ns); pt.s_start.alloc(ns);
    LAUNCH(k_seg_unpack, grid_for(ns, 256), 256, 0, vals.ptr, ns, AT.p.ptr, pt.s_row.ptr, pt.s_len.ptr, pt.s_start.ptr);
}

// one lane per row, natural order: rows of <= SMALL_ROW entries are finished here, rows longer than LONG_ROW are zero-filled
// (their segments arrive through RED.OR), everything in between is left to k_pull_seg.  This kernel is latency-bound, not
// L1TEX-bound: splitting the record across lanes as k_pull_seg does would divide the bytes each warp keeps in flight, so one lane
// owns the whole record here.  ACC (union hops): Y already holds earlier operands' products; small rows are ORed into it and long
// rows are left as they are.
template <int W, bool HINTS, bool ACC>
__global__ void __launch_bounds__(256)
k_pull_small(const u64 *__restrict__ ATp, const u32 *__restrict__ ATj, u64 n, const u64 *__restrict__ X,
             u64 *__restrict__ Y, PullHints ph) {
    const u64 keep = HINTS ? ph.gather_policy(X) : 0, strm = HINTS ? ph.stream_policy() : 0;
    u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    // three-stage pipeline per lane: row pointers two rows ahead, first col_idx batch one row ahead, gathers now
    u64 s = 0, e = 0, s1 = 0, e1 = 0;
    if (j < n) { s = ld_ptr<HINTS>(ATp + j, strm); e = ld_ptr<HINTS>(ATp + j + 1, strm); }
    if (j + stride < n) { s1 = ld_ptr<HINTS>(ATp + j + stride, strm); e1 = ld_ptr<HINTS>(ATp + j + stride + 1, strm); }
    u32 k[4];
#pragma unroll
    for (int u = 0; u < 4; u++) k[u] = (e - s <= SMALL_ROW && s + u < e) ? ld_col<HINTS>(ATj + s + u, strm) : 0xFFFFFFFFu;
    for (; j < n; j += stride) {
        u64 s2 = 0, e2 = 0;
        if (j + 2 * stride < n) { s2 = ld_ptr<HINTS>(ATp + j + 2 * stride, strm); e2 = ld_ptr<HINTS>(ATp + j + 2 * stride + 1, strm); }
        u32 kn[4];
#pragma unroll
        for (int u = 0; u < 4; u++) kn[u] = (e1 - s1 <= SMALL_ROW && s1 + u < e1) ? ld_col<HINTS>(ATj + s1 + u, strm) : 0xFFFFFFFFu;
        u64 acc[W];
#pragma unroll
        for (int w = 0; w < W; w++) acc[w] = 0;
        if (e - s <= SMALL_ROW) {
#pragma unroll
            for (int u = 0; u < 4; u++)
                if (k[u] != 0xFFFFFFFFu) or_words<W, HINTS>(acc, X + (u64)k[u] * W, keep);
            if (e - s > 4) {
#pragma unroll
                for (int u = 0; u < 4; u++) k[u] = (s + 4 + u < e) ? ld_col<HINTS>(ATj + s + 4 + u, strm) : 0xFFFFFFFFu;
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (k[u] != 0xFFFFFFFFu) or_words<W, HINTS>(acc, X + (u64)k[u] * W, keep);
            }
        }
        if (ACC) { if (e - s <= SMALL_ROW) or_part<W>(Y + j * W, acc); }
        else if (e - s <= SMALL_ROW || e - s > LONG_ROW) store_row<W, HINTS>(Y + j * W, acc, strm);
#pragma unroll
        for (int u = 0; u < 4; u++) k[u] = kn[u];
        s = s1; e = e1; s1 = s2; e1 = e2;
    }
}

// 8 lanes per list entry (a mid row, or one LONG_ROW-entry segment of a long row); entries sorted by length, descending.
// Three-stage software pipeline: list entry two steps ahead, col_idx batch one step ahead, gathers now.  Step t of group g
// handles list entry t * ngroups + g on even steps and t * ngroups + (ngroups - 1 - g) on odd ones, which evens out the totals per
// group.  The 8 lanes cover VG vertices x SPLIT record parts per unroll step.  ACC (union hops): a mid row is ORed into the stored
// record instead of replacing it (long-row segments merge with RED.OR either way).
template <int W, bool HINTS, int U, bool EARLY, bool ACC>
__global__ void __launch_bounds__(256)
k_pull_seg(const u32 *__restrict__ s_row, const u64 *__restrict__ s_start, const u32 *__restrict__ s_len, u64 ns,
           const u32 *__restrict__ ATj, const u64 *__restrict__ X, u64 *__restrict__ Y, const u64 *__restrict__ Gp,
           PullHints ph) {
    constexpr int WL = PullCfg<W>::WL, SPLIT = PullCfg<W>::SPLIT, VG = PullCfg<W>::VG;
    const u32 lane8 = threadIdx.x & 7;
    const u32 sub = (threadIdx.x & 31) >> 3;
    const u32 gmask = 0xFFu << (8 * sub);
    const u32 vi = lane8 / SPLIT, h = lane8 % SPLIT;
    const u64 *Xh = X + h * WL;
    const u64 keep = HINTS ? ph.gather_policy(X) : 0, strm = HINTS ? ph.stream_policy() : 0;
    u64 G[WL];
#pragma unroll
    for (int w = 0; w < WL; w++) G[w] = (EARLY && Gp) ? Gp[h * WL + w] : ~0ULL;
    const u64 ngroups = ((u64)gridDim.x * blockDim.x) >> 3;
    const u64 g = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
    const u64 steps = (ns + ngroups - 1) / ngroups;
    auto entry = [&](u64 t) -> u64 { return t * ngroups + ((t & 1) ? ngroups - 1 - g : g); };
    auto fetch = [&](u64 t, u64 &s, u64 &e) {
        s = 0; e = 0;
        if (t < steps) {
            u64 i = entry(t);
            if (i < ns) {   // each entry is fetched once: with hints its lines skip L1
                s = HINTS ? ld_nc_once_u64(s_start + i, strm) : s_start[i];
                e = s + ((HINTS ? ld_nc_once_u32(s_len + i, strm) : s_len[i]) & ~SEG_ATOMIC);
            }
        }
    };
    u64 s0, e0, s1, e1;
    fetch(0, s0, e0);
    fetch(1, s1, e1);
    u32 k[U];
#pragma unroll
    for (int u = 0; u < U; u++) { u64 q = s0 + vi + VG * u; k[u] = (q < e0) ? ld_col<HINTS>(ATj + q, strm) : 0xFFFFFFFFu; }
    for (u64 t = 0; t < steps; t++) {
        u64 s2, e2;
        fetch(t + 2, s2, e2);
        u64 acc[WL];
#pragma unroll
        for (int w = 0; w < WL; w++) acc[w] = 0;
        u64 qb = s0;
        u32 it = 0;
        while (true) {
            const bool more = qb + VG * U < e0;
            const u64 nb = more ? qb + VG * U : s1, ne = more ? e0 : e1;
            u32 kn[U];
#pragma unroll
            for (int u = 0; u < U; u++) { u64 q = nb + vi + VG * u; kn[u] = (q < ne) ? ld_col<HINTS>(ATj + q, strm) : 0xFFFFFFFFu; }
#pragma unroll
            for (int u = 0; u < U; u++)
                if (k[u] != 0xFFFFFFFFu) or_words<WL, HINTS>(acc, Xh + (u64)k[u] * W, keep);
#pragma unroll
            for (int u = 0; u < U; u++) k[u] = kn[u];
            if (!more) break;
            if (EARLY) {   // stop once the entry holds the OR monoid's terminal value: cheap per-lane test, exact cross-lane OR every 4th
                bool full = true;
                if ((it & 3) == 3) {
#pragma unroll
                    for (int w = 0; w < WL; w++) {
                        u64 a = acc[w];
#pragma unroll
                        for (int d = SPLIT; d < 8; d <<= 1) a |= __shfl_xor_sync(gmask, a, d);
                        acc[w] = a;
                        full = full && (a == G[w]);
                    }
                } else {
#pragma unroll
                    for (int w = 0; w < WL; w++) full = full && (acc[w] == G[w]);
                }
                full = __all_sync(gmask, full);
                if (full) {
#pragma unroll
                    for (int u = 0; u < U; u++) { u64 q = s1 + vi + VG * u; k[u] = (q < e1) ? ld_col<HINTS>(ATj + q, strm) : 0xFFFFFFFFu; }
                    break;
                }
            }
            qb += VG * U;
            it++;
        }
#pragma unroll
        for (int w = 0; w < WL; w++) {
            u64 a = acc[w];
#pragma unroll
            for (int d = SPLIT; d < 8; d <<= 1) a |= __shfl_xor_sync(gmask, a, d);
            acc[w] = a;
        }
        if (e0 > s0 && vi == 0) {
            const u64 i = entry(t);
            u64 *dst = Y + (u64)(HINTS ? ld_nc_once_u32(s_row + i, strm) : s_row[i]) * W + h * WL;
            if ((HINTS ? ld_nc_once_u32(s_len + i, strm) : s_len[i]) & SEG_ATOMIC) {
#pragma unroll
                for (int w = 0; w < WL; w++) if (acc[w]) atomicOr((unsigned long long *)(dst + w), acc[w]);
            } else if (ACC) or_part<WL>(dst, acc);
            else store_part<WL, HINTS>(dst, acc, strm);
        }
        s0 = s1; e0 = e1; s1 = s2; e1 = e2;
    }
}

// ---- hot-set packing of the gather index space ------------------------------------------------------------------
// The pull gathers X[k] with k distributed like the out-degree of k.  Relabel k -> slot, slots ordered by out-degree
// descending and restricted to vertices that have out-edges at all (sinks are never gathered): the hot part of the
// frontier words becomes contiguous (L1/L2 resident), and the gather footprint shrinks from 8*W*n to 8*W*n1 bytes.
// shuffle (measurement, hot_shuffle): vertices with out-edges in the order of a hash of their id instead, so the gather
// source has no hot prefix at all; sinks stay last either way
__global__ void k_degree_keys(const u64 *__restrict__ Ap, u64 n, u64 *__restrict__ keys, u64 *__restrict__ n1, bool shuffle) {
    u64 v = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    u64 cnt = 0;
    for (; v < n; v += stride) {
        u64 d = Ap[v + 1] - Ap[v];
        if (d > 0xFFFFFFFEULL) d = 0xFFFFFFFEULL;
        u64 hi = 0xFFFFFFFFULL - d;
        if (shuffle && d) { u32 h = (u32)v * 0x9E3779B1u; h ^= h >> 15; h *= 0x85EBCA77u; h ^= h >> 13; hi = h >> 1; }
        keys[v] = (hi << 32) | v;   // ascending sort => degree descending, then vertex id ascending
        cnt += d != 0;
    }
    if (cnt) atomicAdd((unsigned long long *)n1, cnt);
}
__global__ void k_slots_from_keys(const u64 *__restrict__ keys, const u64 *__restrict__ Ap, u64 n, u64 n1, u32 *__restrict__ vert,
                                  u32 *__restrict__ slot, u32 *__restrict__ hdeg) {
    u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; s < n; s += stride) {
        u32 v = (u32)(keys[s] & 0xFFFFFFFFULL);
        if (s < n1) {
            const u64 d = Ap[v + 1] - Ap[v];
            vert[s] = v; slot[v] = (u32)s; hdeg[s] = d > 0xFFFFFFFEULL ? 0xFFFFFFFEu : (u32)d;
        } else slot[v] = 0xFFFFFFFFu;
    }
}
__global__ void k_full_order(const u64 *__restrict__ keys, u64 n, u32 *__restrict__ pvert, u32 *__restrict__ pperm) {
    u64 s = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; s < n; s += stride) { const u32 v = (u32)(keys[s] & 0xFFFFFFFFULL); pvert[s] = v; pperm[v] = (u32)s; }
}
__global__ void k_relabel_cols(const u32 *__restrict__ j, u64 nnz, const u32 *__restrict__ slot, u32 *__restrict__ jp) {
    u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; q < nnz; q += stride) jp[q] = slot[j[q]];
}
template <int W>
__global__ void k_pack_frontier(const u32 *__restrict__ vert, u64 n1, const u64 *__restrict__ X, u64 *__restrict__ Xp) {
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u64 stride = (u64)gridDim.x * blockDim.x;
    for (; t < n1 * W; t += stride) {
        u64 s = t / W, w = t % W;
        Xp[t] = X[(u64)vert[s] * W + w];
    }
}

// pack + flops + edges + OR-of-everything in one pass over the frontier (fused_prep): the hot set holds every vertex with
// out-edges, so flops = sum popc(X[v]) * deg(v) and edges = sum [X[v] != 0] * deg(v) over it are the exact totals, and
// G[w] = OR of word column w is the terminal value the pull kernels vote against.  One thread per packed word.
template <int W>
__global__ void __launch_bounds__(256)
k_pack_flops(const u32 *__restrict__ vert, const u32 *__restrict__ hdeg, u64 n1, const u64 *__restrict__ X, u64 *__restrict__ Xp,
             u64 *__restrict__ st /* [0] flops [1] edges */, u64 *__restrict__ G) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    __shared__ u64 sG[W];
    if (threadIdx.x < W) sG[threadIdx.x] = 0;
    __syncthreads();
    const u32 lane = threadIdx.x & 31;
    const u32 gmask = (W >= 32) ? 0xffffffffu : (((1u << W) - 1u) << (lane / W * W));   // the W lanes of one vertex
    u64 fl = 0, ed = 0, g = 0;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x, total = n1 * W;
    for (u64 base = t - lane; base < total; base += stride) {       // warp-uniform trip count (ballot inside)
        const u64 tt = base + lane;
        u64 x = 0;
        u32 d = 0;
        if (tt < total) {
            const u64 s = tt / W, w = tt % W;
            x = X[(u64)vert[s] * W + w];
            d = hdeg[s];
            Xp[tt] = x;
        }
        const u32 nz = __ballot_sync(0xffffffffu, x != 0) & gmask;
        fl += (u64)__popcll(x) * d;
        if (nz && (lane % W) == 0) ed += d;
        g |= x;
    }
    // OR across the lanes that hold the same word column (lane % W), then one shared atomic per column and warp
#pragma unroll
    for (int o = W; o < 32; o <<= 1) g |= __shfl_xor_sync(0xffffffffu, g, o);
    if (lane < W && g) atomicOr((unsigned long long *)&sG[lane], g);
    u64 tf = Red(ts).Sum(fl);
    __syncthreads();
    u64 te = Red(ts).Sum(ed);
    if (threadIdx.x == 0) {
        if (tf) atomicAdd((unsigned long long *)&st[0], tf);
        if (te) atomicAdd((unsigned long long *)&st[1], te);
    }
    __syncthreads();
    if (threadIdx.x < W && sG[threadIdx.x]) atomicOr((unsigned long long *)&G[threadIdx.x], sG[threadIdx.x]);
}

// the same totals for a frontier that already IS in hot-set order (permuted form): nothing to gather, nothing to write
template <int W>
__global__ void __launch_bounds__(256)
k_ordered_flops(const u32 *__restrict__ hdeg, u64 n1, const u64 *__restrict__ Xp, u64 *__restrict__ st, u64 *__restrict__ G) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    __shared__ u64 sG[W];
    if (threadIdx.x < W) sG[threadIdx.x] = 0;
    __syncthreads();
    const u32 lane = threadIdx.x & 31;
    const u32 gmask = (W >= 32) ? 0xffffffffu : (((1u << W) - 1u) << (lane / W * W));
    u64 fl = 0, ed = 0, g = 0;
    u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 stride = (u64)gridDim.x * blockDim.x, total = n1 * W;
    for (u64 base = t - lane; base < total; base += stride) {
        const u64 tt = base + lane;
        u64 x = 0;
        u32 d = 0;
        if (tt < total) { x = Xp[tt]; d = hdeg[tt / W]; }
        const u32 nz = __ballot_sync(0xffffffffu, x != 0) & gmask;
        fl += (u64)__popcll(x) * d;
        if (nz && (lane % W) == 0) ed += d;
        g |= x;
    }
#pragma unroll
    for (int o = W; o < 32; o <<= 1) g |= __shfl_xor_sync(0xffffffffu, g, o);
    if (lane < W && g) atomicOr((unsigned long long *)&sG[lane], g);
    u64 tf = Red(ts).Sum(fl);
    __syncthreads();
    u64 te = Red(ts).Sum(ed);
    if (threadIdx.x == 0) {
        if (tf) atomicAdd((unsigned long long *)&st[0], tf);
        if (te) atomicAdd((unsigned long long *)&st[1], te);
    }
    __syncthreads();
    if (threadIdx.x < W && sG[threadIdx.x]) atomicOr((unsigned long long *)&G[threadIdx.x], sG[threadIdx.x]);
}

static void build_hot_pack(const DevCSR &A, const DevCSR &AT, PullTables &pt) {
    u64 n = A.nrows;
    pt.vert.release(); pt.jp.release(); pt.ap.release(); pt.ap_sorted = false; pt.slot.release(); pt.hdeg.release(); pt.n1 = 0; pt.packed = false;
    if (n == 0 || AT.nnz == 0 || n >= 0xFFFFFFFFULL) return;
    DevBuf<u64> keys(n), cnt(1);
    cnt.zero();
    LAUNCH(k_degree_keys, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, A.p.ptr, n, keys.ptr, cnt.ptr, ctx().opt_hot_shuffle != 0);
    sort_keys_u64(keys.ptr, n, 64);
    u64 n1 = read_scalar(cnt.ptr);
    pt.n1 = n1;
    pt.vert.alloc(n1 ? n1 : 1);
    pt.slot.alloc(n);
    pt.hdeg.alloc(n1 ? n1 : 1);
    LAUNCH(k_slots_from_keys, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, keys.ptr, A.p.ptr, n, n1, pt.vert.ptr, pt.slot.ptr, pt.hdeg.ptr);
    // the order over ALL vertices (the sort already put the sinks last, by id): frontiers may be stored in it (permuted form)
    pt.pvert = std::make_shared<DevBuf<u32>>(n);
    pt.pperm = std::make_shared<DevBuf<u32>>(n);
    LAUNCH(k_full_order, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, keys.ptr, n, pt.pvert->ptr, pt.pperm->ptr);
    static std::atomic<u64> next_tag{1};
    pt.perm_tag = next_tag.fetch_add(1);
    pt.packed = true;
}

// The pull tables of one matrix, built once per immutable base (B200_Matrix_prepare, or the first hop that pulls): the hot-set order
// when hot_pack is on, A'.col_idx and A.col_idx relabelled to it, and the segment list.  Turning hot_pack on after the tables
// were built without it adds the order and both relabelled col_idx arrays.
static void build_pull_tables(const DevCSR &A, const DevCSR &AT, PullTables &pt) {
    if (!pt.packed && ctx().opt_hot_pack) build_hot_pack(A, AT, pt);
    if (pt.packed && !pt.jp.ptr) {
        pt.jp.alloc(AT.nnz);
        LAUNCH(k_relabel_cols, grid_for(AT.nnz, 256, (u64)ctx().num_sms * 32), 256, 0, AT.j.ptr, AT.nnz, pt.slot.ptr, pt.jp.ptr);
    }
    // the CSR push's operand: A.col_idx already in the order it writes Y (4 * nnz(A) bytes), so a pushed flop needs no
    // dependent pperm[col] read from a table larger than L2.  Only when perm_push can read it; turning perm_push on later adds
    // it at the next build (until then the push reads pperm[col])
    if (pt.packed && !pt.ap.ptr && ctx().opt_perm_push && A.nnz && A.nrows == A.ncols) {
        pt.ap.alloc(A.nnz);
        LAUNCH(k_relabel_cols, grid_for(A.nnz, 256, (u64)ctx().num_sms * 32), 256, 0, A.j.ptr, A.nnz, pt.pperm->ptr, pt.ap.ptr);
    }
    // its rows ascending by position, for the sliced push (csr_push_sliced): OR commutes and only the CSR push reads ap, so the
    // order inside a row changes no result.  Like ap itself, added at the next build when push_slices was off at the first
    if (pt.ap.ptr && !pt.ap_sorted && ctx().opt_push_slices != 0 && A.nnz <= 0x7fffffffULL) {
        sort_rows_u32(A.p.ptr, A.nrows, pt.ap.ptr, A.nnz);
        pt.ap_sorted = true;
    }
    if (!pt.built) {
        build_seg_list(AT, pt);
        pt.built = true;
    }
}

// every CTA of a 256-thread kernel that can be resident at once: occupancy x SMs, at least one CTA per SM
template <class K> static u64 full_wave(K kern) {
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, 0));
    return (u64)ctx().num_sms * (u64)std::max(per_sm, 1);
}

// k_pull_small over every row of A', then k_pull_seg over the segment list.  The segment kernel's grid is every CTA resident at
// once (occupancy x SMs) unless pull_grid overrides it: entries are dealt round-robin to 8-lane groups, so one full wave keeps all
// SMs busy to the end.
template <int W, bool HINTS, bool ACC>
static void launch_pull(const DevCSR &AT, const PullTables &pt, u64 m, const u32 *gj, const u64 *gx, u64 *Y, const u64 *Gp,
                        PullHints ph) {
    Context &cx = ctx();
    LAUNCH((k_pull_small<W, HINTS, ACC>), grid_for(m, 256, (u64)cx.num_sms * 32), 256, 0, AT.p.ptr, gj, m, gx, Y, ph);
    if (!pt.ns) return;
    auto seg = [&](auto kern) {
        const u64 grid = cx.opt_pull_grid > 0 ? (u64)cx.num_sms * (u64)cx.opt_pull_grid : full_wave(kern);
        LAUNCH(kern, (u32)grid, 256, 0, pt.s_row.ptr, pt.s_start.ptr, pt.s_len.ptr, pt.ns, gj, gx, Y, Gp, ph);
    };
    if (Gp) seg(k_pull_seg<W, HINTS, 4, true, ACC>);
    else seg(k_pull_seg<W, HINTS, 4, false, ACC>);
}

// The pull's L2 policies, as measured on the H100 (scripts/pull_l2.py, DESIGN §4.8): from W = 2 up, the first half of the L2 of
// the gather source is evict_last and the rest evict_first (0.41 ms off a 4.6 ms W = 8 pull); the streams are evict_first only at
// W = 2 and 4, where that gains another 0.08 ms -- at W = 8 and 16 it costs 0.07-0.16 ms.  At W = 1 no policy pays.
// The prefix never exceeds the source.  (createpolicy.range takes 32-bit sizes: a source past 4 GB has its first 4 GB in the range.)
static bool pull_hints_on(int W) { const i64 o = ctx().opt_hints; return o > 0 || (o < 0 && W >= 2); }
static PullHints pull_hints(int W, u64 x_bytes) {
    const Context &cx = ctx();
    PullHints ph;
    ph.tot = x_bytes > 0xFFFFFFF0ULL ? 0xFFFFFFF0u : (u32)x_bytes;
    const u64 hot = cx.opt_hot_bytes >= 0 ? (u64)cx.opt_hot_bytes : cx.l2_bytes / 2;
    ph.hot = hot < ph.tot ? (u32)hot : ph.tot;
    ph.streams = cx.opt_hint_streams >= 0 ? cx.opt_hint_streams != 0 : (W == 2 || W == 4);
    return ph;
}

template <int W>
static void hop_impl(const DevBits &Xin, const DevCSR &A, const DevCSR *AT, PullTables *pt, DevBits &Y,
                     u64 *flops_out, int *path_out, bool acc) {
    Context &cx = ctx();
    u64 n = A.nrows, m = A.ncols;
    // X in permuted form: usable as it stands only by the pull through the tables it was ordered for; anything else works on a
    // natural-order copy (cannot happen on the bench path: the caller orders a frontier only for the operand it is pushed through)
    DevBits Xnat;
    const bool ordered = Xin.permuted() && AT && pt && pt->packed && Xin.perm_tag == pt->perm_tag && pt->jp.ptr && pt->hdeg.ptr &&
                         cx.opt_pull_mode != 0 && cx.opt_hot_pack && n == m;
    const DevBits *Xuse = &Xin;
    if (Xin.permuted() && !ordered) { bits_copy(Xin, Xnat); bits_naturalise(Xnat); Xuse = &Xnat; }
    const DevBits &X = *Xuse;
    if (!acc) {
        Y.clear();
        Y.nrows = X.nrows; Y.ncols = m; Y.W = W;
        Y.w.alloc(m * W);
    }
    DevBuf<u32> flag(n + 1);
    DevBuf<u64> st(2);
    st.zero();
    // fused_prep: when the hot-set tables exist, one pass packs the frontier for the pull AND yields flops / edges / the OR
    // terminal; the separate flops pass (needed for its per-vertex flags) then only runs if the push direction wins
    const bool fused = cx.opt_fused_prep && AT && pt && cx.opt_hot_pack && pt->packed && pt->jp.ptr && pt->hdeg.ptr &&
                       cx.opt_pull_mode != 0 && n == m;
    DevBuf<u64> Xp, Gd;
    if (ordered) {            // already in gather order: totals only
        Gd.alloc(W);
        Gd.zero();
        if (pt->n1) LAUNCH((k_ordered_flops<W>), grid_for(pt->n1 * W, 256, (u64)ctx().num_sms * 16), 256, 0, pt->hdeg.ptr, pt->n1, X.w.ptr, st.ptr, Gd.ptr);
    } else if (fused) {
        Xp.alloc(pt->n1 * W);
        Gd.alloc(W);
        Gd.zero();
        if (pt->n1) LAUNCH((k_pack_flops<W>), grid_for(pt->n1 * W, 256, (u64)ctx().num_sms * 16), 256, 0, pt->vert.ptr, pt->hdeg.ptr, pt->n1, X.w.ptr, Xp.ptr, st.ptr, Gd.ptr);
    } else if (n) LAUNCH(k_bits_flops, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, X.w.ptr, (u32)W, n, A.p.ptr, flag.ptr, st.ptr);
    u64 hst[2] = {0, 0};
    d2h(hst, st.ptr, 2);
    sync_stream();
    if (flops_out) *flops_out = hst[0];
    u64 edges = hst[1];
    bool pull = false;
    if (AT && pt) {
        if (cx.opt_pull_mode == 1) pull = true;
        else if (cx.opt_pull_mode == 0) pull = false;
        else pull = edges * 4 > A.nnz; // direction switch: frontier touches > 1/4 of the edges
    }
    if (edges == 0) { if (!acc) Y.w.zero(); if (path_out) *path_out = 0; return; }
    if (ordered && !pull) {                     // the push direction works on natural order: undo the frontier's order and start over
        DevBits Xn;
        bits_copy(Xin, Xn);
        bits_naturalise(Xn);
        hop_impl<W>(Xn, A, AT, pt, Y, flops_out, path_out, acc);
        return;
    }
    if (!pull) {
        if (fused) {                            // push needs the per-vertex active flags of the classic pass
            DevBuf<u64> st2(2);
            st2.zero();
            LAUNCH(k_bits_flops, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, X.w.ptr, (u32)W, n, A.p.ptr, flag.ptr, st2.ptr);
        }
        if (!acc) Y.w.zero();                   // accumulate: the REDs OR into the earlier operands' product
        CUDA_TRY(cudaMemsetAsync(flag.ptr + n, 0, sizeof(u32), stream()));
        DevBuf<u64> pos(n + 1);
        exclusive_scan_u32_to_u64(flag.ptr, pos.ptr, n + 1);
        u64 nact = read_scalar(pos.ptr + n);
        DevBuf<u32> act(nact);
        DevBuf<u64> cum(nact + 1), astart(nact);
        LAUNCH(k_compact_active, grid_for(n, 256, 1 << 16), 256, 0, flag.ptr, pos.ptr, n, A.p.ptr, act.ptr, cum.ptr, astart.ptr);
        CUDA_TRY(cudaMemsetAsync(cum.ptr + nact, 0, sizeof(u64), stream()));
        exclusive_scan_u64(cum.ptr, cum.ptr, nact + 1);
        u64 nchunks = (edges + PUSH_CHUNK - 1) / PUSH_CHUNK;
        {
            // col_idx segments + per-active (id,cum,start) + X words + one RED per (edge, word); the same bytes when accumulating
            TimedScope ts(acc ? TK_BITS_PUSH_ACC : TK_BITS_PUSH, 4 * edges + 20 * nact + 8ULL * W * nact + 8ULL * W * edges);
            LAUNCH((k_bits_push<W>), (u32)nchunks, 256, 0, act.ptr, cum.ptr, astart.ptr, nact, edges, A.j.ptr, X.w.ptr, Y.w.ptr);
        }
        if (path_out) *path_out = 2;
        return;
    }
    build_pull_tables(A, *AT, *pt);             // a no-op once the matrix has them
    const u32 *gj = AT->j.ptr;                  // gather index stream
    const u64 *gx = X.w.ptr;                    // gather source
    u64 gn = n;                                 // gather footprint in vertices
    if (ordered) {                              // the frontier already is the packed gather source (its first n1 records)
        gj = pt->jp.ptr; gx = X.w.ptr; gn = pt->n1;
    } else if (cx.opt_hot_pack && pt->packed) {
        if (!fused) {
            Xp.alloc(pt->n1 * W);
            if (pt->n1) LAUNCH((k_pack_frontier<W>), grid_for(pt->n1 * W, 256, (u64)ctx().num_sms * 32), 256, 0, pt->vert.ptr, pt->n1, X.w.ptr, Xp.ptr);
        }
        gj = pt->jp.ptr; gx = Xp.ptr; gn = pt->n1;
    }
    const u64 *Gp = nullptr;
    // opt_early_exit: 0 never, 1 auto, 2 always.  Auto: the in-loop vote pays for itself at W = 2 and 4 (hub rows saturate),
    // costs more than it saves at W = 1 (few rows ever hold all 64 bits) and at W >= 8; very dense frontiers always benefit.
    const bool dense_frontier = hst[0] >= (hst[1] * X.nrows) / 4;   // flops/edges = degree-weighted mean popcount of a gathered word
    if (cx.opt_early_exit == 2 || (cx.opt_early_exit == 1 && (dense_frontier || W == 2 || W == 4))) {
        if (!((fused && gx == Xp.ptr) || ordered)) {   // the fused / ordered pass already left the OR of the packed frontier in Gd
            Gd.alloc(W);
            Gd.zero();
            if (gn) LAUNCH((k_or_all<W>), grid_for(gn, 256, (u64)ctx().num_sms * 8), 256, 0, gx, gn, Gd.ptr);
        }
        Gp = Gd.ptr;
    }
    {
        // compulsory traffic: stream A' col_idx + rowptr, read X once, write Y once (X gathers hit L2).  Accumulating ("bits_pull_acc"),
        // Y is also read once: an upper bound, rows with nothing to add skip the read and the write.
        TimedScope ts(acc ? TK_BITS_PULL_ACC : TK_BITS_PULL, 4 * AT->nnz + 8 * (m + 1) + 8ULL * W * gn + (acc ? 16ULL : 8ULL) * W * m);
        const PullHints ph = pull_hints(W, gn * W * 8);
        const bool hints = pull_hints_on(W);
        if (acc) {
            if (hints) launch_pull<W, true, true>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
            else launch_pull<W, false, true>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
        } else if (hints) launch_pull<W, true, false>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
        else launch_pull<W, false, false>(*AT, *pt, m, gj, gx, Y.w.ptr, Gp, ph);
    }
    if (path_out) *path_out = 3;
}

// builds the pull tables of a square operand now (B200_Matrix_prepare) instead of inside the first hop that pulls
void bits_prepare_pull(const DevCSR &A, const DevCSR &AT, PullTables &pt) {
    if (A.nrows != A.ncols || !AT.nnz) return;
    build_pull_tables(A, AT, pt);
}

void bits_hop(const DevBits &X, const DevCSR &A, const DevCSR *AT, PullTables *pt, DevBits &Y, u64 *flops_out,
              int *path_out, bool acc) {
    if (X.ncols != A.nrows) throw GrbError(-6, "mxm: inner dimensions differ");
    if (acc) require_acc_target(Y, X.nrows, A.ncols, X.W);
    with_words(X.W, [&](auto w) { hop_impl<w>(X, A, AT, pt, Y, flops_out, path_out, acc); });
}

// ---------------------------------------------------------------------------- exact dirty hop (reach over (m \ dm) u dp)
// delta_lmxm's AND-NOT term over-masks: it drops (i, j) whenever ANY deleted edge reaches j from row i, even when a remaining edge
// still reaches it.  A reach over a tensor with pending deletions needs X * (m \ dm) exactly.  Only the columns dm touches can
// differ from X * m, so those columns are recomputed: Y[pos(j)] = OR of X[pos(k)] over the in-edges k of m'(j, :) that are not in
// dm'(j, :).  Both rows are sorted, so a lane finds its in-edge in the deleted list with a lower bound that only moves forward.
// Hub columns are cut into REPAIR_SEG-entry segments, as the pull cuts long rows: a column of several segments is zeroed first and
// its segments arrive through RED.OR; a column of one segment is stored.  Work is O(W * the repaired columns' in-degrees).
static const u64 REPAIR_SEG = 1024;
static const u32 REPAIR_ATOMIC = 0x80000000u, REPAIR_FIRST = 0x40000000u, REPAIR_LEN = 0x3FFFFFFFu;

// segments per column: ceil(indeg_m(j) / REPAIR_SEG) where dm' has a row j, else 0;  st = {repaired columns, their in-edges}
__global__ void __launch_bounds__(256)
k_repair_count(const u64 *__restrict__ Dp, const u64 *__restrict__ Tp, u64 n, u32 *__restrict__ cnt, u64 *__restrict__ st) {
    typedef cub::BlockReduce<u64, 256> Red;
    __shared__ typename Red::TempStorage ts;
    u64 c = 0, e = 0;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j <= n; j += stride) {
        if (j == n) { cnt[j] = 0; continue; }
        const u64 d = Dp[j + 1] > Dp[j] ? Tp[j + 1] - Tp[j] : 0;
        cnt[j] = (u32)((d + REPAIR_SEG - 1) / REPAIR_SEG);
        c += d != 0;
        e += d;
    }
    const u64 tc = Red(ts).Sum(c);
    __syncthreads();
    const u64 te = Red(ts).Sum(e);
    if (threadIdx.x == 0) {
        if (tc) atomicAdd((unsigned long long *)&st[0], tc);
        if (te) atomicAdd((unsigned long long *)&st[1], te);
    }
}
__global__ void k_repair_emit(const u64 *__restrict__ Tp, const u32 *__restrict__ cnt, const u64 *__restrict__ pos, u64 n,
                              u32 *__restrict__ s_col, u64 *__restrict__ s_start, u32 *__restrict__ s_len) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
        const u32 c = cnt[j];
        if (!c) continue;
        const u64 t0 = Tp[j], d = Tp[j + 1] - t0, o = pos[j];
        for (u32 i = 0; i < c; i++) {
            const u64 s = (u64)i * REPAIR_SEG, len = d - s < REPAIR_SEG ? d - s : REPAIR_SEG;
            s_col[o + i] = (u32)j;
            s_start[o + i] = t0 + s;
            s_len[o + i] = (u32)len | (c > 1 ? (REPAIR_ATOMIC | (i == 0 ? REPAIR_FIRST : 0u)) : 0u);
        }
    }
}
// the columns merged with RED.OR start from zero (their first segment names them once)
template <int W>
__global__ void k_repair_zero(const u32 *__restrict__ s_col, const u32 *__restrict__ s_len, u64 ns, const u32 *__restrict__ yperm,
                              u64 *__restrict__ Y) {
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += stride) {
        if (!(s_len[i] & REPAIR_FIRST)) continue;
        const u64 j = s_col[i], py = yperm ? yperm[j] : j;
#pragma unroll
        for (int w = 0; w < W; w++) Y[py * W + w] = 0;
    }
}
// 8 lanes per segment, dealt round-robin; inside a group VG in-edges x SPLIT record parts per unroll step (the pull's lane split).
template <int W, int U>
__global__ void __launch_bounds__(256)
k_bits_repair(const u32 *__restrict__ s_col, const u64 *__restrict__ s_start, const u32 *__restrict__ s_len, u64 ns,
              const u32 *__restrict__ Tj, const u64 *__restrict__ Dp, const u32 *__restrict__ Dj, const u64 *__restrict__ X,
              const u32 *__restrict__ xperm, u64 *__restrict__ Y, const u32 *__restrict__ yperm) {
    constexpr int WL = PullCfg<W>::WL, SPLIT = PullCfg<W>::SPLIT, VG = PullCfg<W>::VG;
    const u32 lane8 = threadIdx.x & 7;
    const u32 gmask = 0xFFu << (8 * ((threadIdx.x & 31) >> 3));
    const u32 vi = lane8 / SPLIT, h = lane8 % SPLIT;
    const u64 *Xh = X + h * WL;
    const u64 ngroups = ((u64)gridDim.x * blockDim.x) >> 3;
    for (u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 3; i < ns; i += ngroups) {   // uniform inside the 8-lane group
        const u32 j = __ldg(s_col + i), fl = __ldg(s_len + i);
        const u64 s = __ldg(s_start + i), e = s + (fl & REPAIR_LEN), de = __ldg(Dp + j + 1);
        u64 d = __ldg(Dp + j);
        u64 acc[WL];
#pragma unroll
        for (int w = 0; w < WL; w++) acc[w] = 0;
        for (u64 qb = s; qb < e; qb += VG * U) {
            u32 k[U];
#pragma unroll
            for (int u = 0; u < U; u++) { const u64 q = qb + vi + VG * u; k[u] = q < e ? __ldg(Tj + q) : 0xFFFFFFFFu; }
#pragma unroll
            for (int u = 0; u < U; u++) {
                if (k[u] == 0xFFFFFFFFu) continue;
                u64 lo = d, hi = de;                 // lower bound of k[u] among the deleted sources of j
                while (lo < hi) {
                    const u64 mid = (lo + hi) >> 1;
                    if (__ldg(Dj + mid) < k[u]) lo = mid + 1; else hi = mid;
                }
                d = lo;
                if (d < de && __ldg(Dj + d) == k[u]) continue;   // a deleted edge
                const u64 px = xperm ? __ldg(xperm + k[u]) : k[u];
                or_words<WL, false>(acc, Xh + px * W, 0);
            }
        }
#pragma unroll
        for (int w = 0; w < WL; w++) {
            u64 a = acc[w];
#pragma unroll
            for (int dd = SPLIT; dd < 8; dd <<= 1) a |= __shfl_xor_sync(gmask, a, dd);
            acc[w] = a;
        }
        if (vi == 0) {
            const u64 py = yperm ? __ldg(yperm + j) : j;
            u64 *dst = Y + py * W + h * WL;
            if (fl & REPAIR_ATOMIC) {
#pragma unroll
                for (int w = 0; w < WL; w++) if (acc[w]) atomicOr((unsigned long long *)(dst + w), acc[w]);
            } else store_part<WL>(dst, acc);
        }
    }
}

void bits_repair_plan(const DevCSR &dm, const DevCSR &mT, RepairPlan &rp) {
    if (dm.nrows != mT.ncols || dm.ncols != mT.nrows) throw GrbError(-6, "reach: delta dimensions differ from the operand");
    rp.ns = rp.ncols = rp.inedges = 0;
    rp.s_col.release(); rp.s_len.release(); rp.s_start.release();
    rp.dmT.clear();
    const u64 n = mT.nrows;
    if (!dm.nnz || !n) return;
    transpose_csr(dm, rp.dmT, false);                  // dm changes with every write: built per call
    DevBuf<u32> cnt(n + 1);
    DevBuf<u64> pos(n + 1), st(2);
    st.zero();
    LAUNCH(k_repair_count, grid_for(n + 1, 256, (u64)ctx().num_sms * 16), 256, 0, rp.dmT.p.ptr, mT.p.ptr, n, cnt.ptr, st.ptr);
    exclusive_scan_u32_to_u64(cnt.ptr, pos.ptr, n + 1);
    u64 h[3];
    d2h(h, st.ptr, 2);
    d2h(h + 2, pos.ptr + n, 1);
    sync_stream();
    rp.ncols = h[0]; rp.inedges = h[1]; rp.ns = h[2];
    if (!rp.ns) return;
    rp.s_col.alloc(rp.ns); rp.s_len.alloc(rp.ns); rp.s_start.alloc(rp.ns);
    LAUNCH(k_repair_emit, grid_for(n, 256, (u64)ctx().num_sms * 16), 256, 0, mT.p.ptr, cnt.ptr, pos.ptr, n, rp.s_col.ptr,
           rp.s_start.ptr, rp.s_len.ptr);
}

template <int W>
static void repair_impl(const DevBits &X, const DevCSR &mT, const RepairPlan &rp, DevBits &Y) {
    const u32 *xperm = pos_table(X), *yperm = pos_table(Y);
    // two row pointers per repaired column, m' and dm' column ids, the gathered records, the stored columns
    TimedScope ts(TK_BITS_REPAIR, 16 * rp.ncols + 4 * rp.inedges + 4 * rp.dmT.nnz + 8ULL * W * rp.inedges + 8ULL * W * rp.ncols);
    LAUNCH((k_repair_zero<W>), grid_for(rp.ns, 256, (u64)ctx().num_sms * 16), 256, 0, rp.s_col.ptr, rp.s_len.ptr, rp.ns, yperm, Y.w.ptr);
    const u64 need = (rp.ns * 8 + 255) / 256, full = full_wave(k_bits_repair<W, 4>);
    LAUNCH((k_bits_repair<W, 4>), (u32)(need < full ? need : full), 256, 0, rp.s_col.ptr, rp.s_start.ptr, rp.s_len.ptr, rp.ns, mT.j.ptr,
           rp.dmT.p.ptr, rp.dmT.j.ptr, X.w.ptr, xperm, Y.w.ptr, yperm);
}

void bits_repair(const DevBits &X, const DevCSR &mT, const RepairPlan &rp, DevBits &Y) {
    if (!rp.ns) return;
    if (X.ncols != mT.ncols || Y.ncols != mT.nrows) throw GrbError(-6, "reach: frontier dimensions differ from the operand");
    if (X.W != Y.W) throw GrbError(-101, "reach: frontier and product word counts differ");
    require_pos_table(Y, "reach");
    require_pos_table(X, "reach");
    with_words(Y.W, [&](auto w) { repair_impl<w>(X, mT, rp, Y); });
}

} // namespace b200
