// writes.cu -- the read phase of a relationship Tensor's batched writes (B200_Tensor_insert_plan / B200_Tensor_remove_plan):
// what Tensor::set_all_from_slices (tensor.rs:333-447) and Tensor::remove_all's multi-edge path (tensor.rs:454-629) decide per edge
// with dp.get / dm.contains / m.get / mt.m / me.m probes on the host, for a whole batch in one pass over the live layers.  The
// host then makes the reference's write calls from the plan and reads no layer.
//
// Insert.  Keys src << 32 | dst with the batch position as value, stable radix sort: a pair's run holds its ids in batch order.
// One thread per run probes dp, dm, m and mt.m (plus me.m for each me entry it emits) and counts the run's inline record (0 / 1)
// and me entries (0, g or g + 1); scans of the counts place them, a fill pass writes them.
// Remove.  (key, id) sorted by two stable radix sorts (id, then key); a run's duplicate ids are adjacent and skipped.  One thread
// per run takes Tensor::eff_get, and for a MULTI_EDGE pair merges the run's ids with the key's merged id list: H = the ids named,
// rem = the rest.  Count, scan and fill as above.  Like edges.cu, one thread walks one pair's id list (twice: count and fill), so
// a pair with very many multi-edges serialises on its thread.
#include "edge_layers.cuh"

namespace b200 {

// a run's kind (insert): the pair's value before the batch
static const uint8_t WK_MULTI = 0, WK_SINGLE = 1, WK_NONE = 2;

// key[k] = src[k] << 32 | dst[k]; val[k] = id[k] (remove), or k, the batch position (insert, id null)
__global__ void k_wp_keys(const u64 *__restrict__ src, const u64 *__restrict__ dst, const u64 *__restrict__ id, u64 n,
                          u64 *__restrict__ key, u64 *__restrict__ val) {
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (u64)gridDim.x * blockDim.x) {
        key[k] = src[k] << 32 | dst[k];
        val[k] = id ? id[k] : k;
    }
}
// rstart[r] = the first position of run r; rstart[R] = n
__global__ void k_wp_starts(const u32 *__restrict__ head, const u64 *__restrict__ hpos, u64 n, u64 *__restrict__ rstart) {
    for (u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x; k <= n; k += (u64)gridDim.x * blockDim.x)
        if (k == n || head[k]) rstart[hpos[k]] = k;
}

// is v among ids[lo, hi) (ascending)
__device__ __forceinline__ bool ids_has(const u64 *__restrict__ ids, u64 lo, u64 hi, u64 v) {
    const u64 q = lb64(ids, lo, hi, v);
    return q < hi && ids[q] == v;
}

// ---- insert plan ----
// per run: the pair's value before the batch (cur), the inline record's value and flags, the record and me entry counts
__global__ void k_ins_count(EType t, const u64 *__restrict__ key, const u64 *__restrict__ pos, const u64 *__restrict__ id,
                            const u64 *__restrict__ rstart, u64 R, u64 *__restrict__ rcur, u64 *__restrict__ rinl,
                            uint8_t *__restrict__ rkind, uint8_t *__restrict__ rflags, u32 *__restrict__ in_cnt,
                            u32 *__restrict__ me_cnt) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (u64)gridDim.x * blockDim.x) {
        const u64 a = rstart[r], g = rstart[r + 1] - a, kk = key[a], s = kk >> 32;
        const u32 d = (u32)kk;
        const u64 qdp = find_rc(t.dp, s, d), qm = find_rc(t.m, s, d);
        const bool masked = find_rc(t.dm, s, d) != ~0ULL, mhas = qm != ~0ULL;
        const u64 mval = mhas ? t.m.x[qm] : 0;
        bool has = false;
        u64 cur = 0;
        if (qdp != ~0ULL) { has = true; cur = t.dp.x[qdp]; }     // set_all_from_slices: dp, else nothing under dm, else m
        else if (!masked) { has = mhas; cur = mval; }
        uint8_t kind, fl = 0;
        u32 nin = 1, nme;
        u64 inl = EE_MULTI;
        bool committed;
        if (has && cur == EE_MULTI) { kind = WK_MULTI; nin = 0; nme = (u32)g; committed = false; }
        else if (has) { kind = WK_SINGLE; nme = (u32)g + 1; committed = qdp != ~0ULL && mhas; }
        else { kind = WK_NONE; nme = g == 1 ? 0 : (u32)g; if (g == 1) inl = id[pos[a]]; committed = masked && mhas; }
        if (nin) {
            if (committed) fl |= WP_COMMITTED;
            if (committed && mval == inl) fl |= WP_CANCEL;
            if (find_rc(t.mt, d, s) != ~0ULL) fl |= WP_MT_BASE;
        }
        rcur[r] = cur; rinl[r] = inl; rkind[r] = kind; rflags[r] = fl;
        in_cnt[r] = nin; me_cnt[r] = nme;
    }
}

__global__ void k_ins_fill(EType t, const u64 *__restrict__ key, const u64 *__restrict__ pos, const u64 *__restrict__ id,
                           const u64 *__restrict__ rstart, u64 R, const u64 *__restrict__ rcur, const u64 *__restrict__ rinl,
                           const uint8_t *__restrict__ rkind, const uint8_t *__restrict__ rflags, const u64 *__restrict__ in_pos,
                           const u64 *__restrict__ me_pos, u64 *__restrict__ o_src, u64 *__restrict__ o_dst, u64 *__restrict__ o_val,
                           uint8_t *__restrict__ o_flags, u64 *__restrict__ o_key, u64 *__restrict__ o_id, uint8_t *__restrict__ o_base) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (u64)gridDim.x * blockDim.x) {
        const u64 a = rstart[r], e = rstart[r + 1], kk = key[a];
        const uint8_t kind = rkind[r];
        if (kind != WK_MULTI) {
            const u64 o = in_pos[r];
            o_src[o] = kk >> 32; o_dst[o] = kk & 0xFFFFFFFFULL; o_val[o] = rinl[r]; o_flags[o] = rflags[r];
        }
        u64 o = me_pos[r];
        if (o == me_pos[r + 1]) continue;
        u64 lo, hi;
        key_range(t.me, kk, &lo, &hi);
        auto put = [&](u64 x) { o_key[o] = kk; o_id[o] = x; o_base[o] = ids_has(t.me.id, lo, hi, x); o++; };
        if (kind == WK_SINGLE) put(rcur[r]);                    // promotion: the inline id first, then the batch's
        for (u64 k = a; k < e; k++) put(id[pos[k]]);
    }
}

// ---- remove plan ----
// per run (ids ascending): the pair record's value and flags, the record and me entry counts
__global__ void k_rm_count(EType t, const u64 *__restrict__ key, const u64 *__restrict__ id, const u64 *__restrict__ rstart, u64 R,
                           u64 *__restrict__ rval, uint8_t *__restrict__ rflags, u32 *__restrict__ pr_cnt, u32 *__restrict__ me_cnt) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (u64)gridDim.x * blockDim.x) {
        const u64 a = rstart[r], e = rstart[r + 1], kk = key[a], s = kk >> 32;
        const u32 d = (u32)kk;
        uint8_t fl = 0;
        u32 nme = 0;
        u64 v = 0;
        if (eff_get(t, s, d, &v)) {
            if (v != EE_MULTI) {
                if (ids_has(id, a, e, v)) fl = WP_EMPTIED;
            } else {
                u64 c = a, nh = 0, nl = 0, surv = 0;
                merged_ids(t, kk, [&](u64, u64 x) {
                    while (c < e && id[c] < x) c++;
                    if (c < e && id[c] == x) nh++; else surv = x;
                    nl++;
                    return true;
                });
                if (nh) {                                       // a list of fewer than two ids (a live id added twice) only
                    const u64 rem = nl - nh;                    // loses the ids named, like the host's walk
                    if (rem >= 2 || nl < 2) nme = (u32)nh;
                    else { nme = (u32)nl; fl = rem ? WP_DEMOTED : WP_EMPTIED; if (rem) v = surv; }
                }
            }
            if (fl) {
                const u64 qm = find_rc(t.m, s, d);
                if (qm != ~0ULL) { fl |= WP_M_HAS; if ((fl & WP_DEMOTED) && t.m.x[qm] == v) fl |= WP_M_EQ; }
                if (find_rc(t.mt, d, s) != ~0ULL) fl |= WP_MT_BASE;
            }
        }
        rval[r] = v; rflags[r] = fl;
        pr_cnt[r] = fl ? 1 : 0; me_cnt[r] = nme;
    }
}

__global__ void k_rm_fill(EType t, const u64 *__restrict__ key, const u64 *__restrict__ id, const u64 *__restrict__ rstart, u64 R,
                          const u64 *__restrict__ rval, const uint8_t *__restrict__ rflags, const u64 *__restrict__ pr_pos,
                          const u64 *__restrict__ me_pos, u64 *__restrict__ o_src, u64 *__restrict__ o_dst, u64 *__restrict__ o_val,
                          uint8_t *__restrict__ o_flags, u64 *__restrict__ o_key, u64 *__restrict__ o_id, uint8_t *__restrict__ o_base) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < R; r += (u64)gridDim.x * blockDim.x) {
        const u64 a = rstart[r], e = rstart[r + 1], kk = key[a];
        const uint8_t fl = rflags[r];
        if (fl) {
            const u64 o = pr_pos[r];
            o_src[o] = kk >> 32; o_dst[o] = kk & 0xFFFFFFFFULL; o_val[o] = rval[r]; o_flags[o] = fl;
        }
        u64 o = me_pos[r];
        if (o == me_pos[r + 1]) continue;
        const bool all = fl != 0;                                // demoted or emptied: the whole list; else the ids named
        u64 lo, hi, c = a;
        key_range(t.me, kk, &lo, &hi);
        merged_ids(t, kk, [&](u64, u64 x) {
            while (c < e && id[c] < x) c++;
            if (all || (c < e && id[c] == x)) { o_key[o] = kk; o_id[o] = x; o_base[o] = ids_has(t.me.id, lo, hi, x); o++; }
            return true;
        });
    }
}

// sort bits of the keys: src < nv <= 2^32
static int key_bits(u64 nv) { int b = 0; while (b < 32 && ((u64)1 << b) < nv) b++; return 32 + b; }

// the runs of equal keys of the sorted key[0 .. n): rstart[0 .. R] (rstart[R] = n); returns R
static u64 mark_runs(const u64 *key, u64 n, u32 grid, DevBuf<u64> &rstart) {
    DevBuf<u32> head(n + 1);
    DevBuf<u64> hpos(n + 1);
    const u64 R = run_heads(key, n, head.ptr, hpos.ptr);
    rstart.alloc(n + 1);
    LAUNCH(k_wp_starts, grid_for(n + 1, 256, grid), 256, 0, head.ptr, hpos.ptr, n, rstart.ptr);
    return R;
}

// the scans of the per-run counts (R + 1 entries, the last 0): positions and the two totals
static void place(const u32 *c1, const u32 *c2, u64 R, DevBuf<u64> &p1, DevBuf<u64> &p2, u64 *n1, u64 *n2) {
    p1.alloc(R + 1); p2.alloc(R + 1);
    exclusive_scan_u32_to_u64(c1, p1.ptr, R + 1);
    exclusive_scan_u32_to_u64(c2, p2.ptr, R + 1);
    d2h(n1, p1.ptr + R, 1);
    d2h(n2, p2.ptr + R, 1);
    sync_stream();
}

// the plan's device arrays, copied to the caller's host arrays
struct PlanBufs {
    DevBuf<u64> src, dst, val, key, id;
    DevBuf<uint8_t> flags, base;
    PlanBufs(u64 nrec, u64 nme) : src(nrec), dst(nrec), val(nrec), key(nme), id(nme), flags(nrec), base(nme) {}
    void to_host(WritePlan &P) {
        d2h(P.rec_src, src.ptr, P.nrec); d2h(P.rec_dst, dst.ptr, P.nrec); d2h(P.rec_val, val.ptr, P.nrec);
        d2h(P.rec_flags, flags.ptr, P.nrec);
        d2h(P.me_key, key.ptr, P.nme); d2h(P.me_id, id.ptr, P.nme); d2h(P.me_base, base.ptr, P.nme);
        sync_stream();
    }
};

void tensor_insert_plan(const EdgeTypeDev &type, const u64 *d_src, const u64 *d_dst, const u64 *d_id, u64 n, u64 nv, WritePlan &P) {
    const EType t = etype(type);
    const u32 grid = (u32)ctx().num_sms * 8;
    DevBuf<u64> key(n), pos(n), rstart;
    // Compulsory bytes ("tensor_write"): 24 per batch edge (src, dst, id read once), 64 per distinct pair (the row pointers of dp,
    // dm, m and mt it probes), 25 per inline record (src, dst, value, flags) and 17 per me entry (key, id, base flag).
    TimedScope ts(TK_TENSOR_WRITE, 0);
    LAUNCH(k_wp_keys, grid_for(n, 256, grid), 256, 0, d_src, d_dst, (const u64 *)nullptr, n, key.ptr, pos.ptr);
    sort_pairs_u64(key.ptr, pos.ptr, n, key_bits(nv));
    const u64 R = mark_runs(key.ptr, n, grid, rstart);
    DevBuf<u64> rcur(R), rinl(R), in_pos, me_pos;
    DevBuf<uint8_t> rkind(R), rflags(R);
    DevBuf<u32> in_cnt(R + 1), me_cnt(R + 1);
    CUDA_TRY(cudaMemsetAsync(in_cnt.ptr + R, 0, sizeof(u32), stream()));
    CUDA_TRY(cudaMemsetAsync(me_cnt.ptr + R, 0, sizeof(u32), stream()));
    LAUNCH(k_ins_count, grid_for(R, 256, grid), 256, 0, t, key.ptr, pos.ptr, d_id, rstart.ptr, R, rcur.ptr, rinl.ptr, rkind.ptr,
           rflags.ptr, in_cnt.ptr, me_cnt.ptr);
    place(in_cnt.ptr, me_cnt.ptr, R, in_pos, me_pos, &P.nrec, &P.nme);
    ts.bytes = 24 * n + 64 * R + 25 * P.nrec + 17 * P.nme;
    PlanBufs out(P.nrec, P.nme);
    LAUNCH(k_ins_fill, grid_for(R, 256, grid), 256, 0, t, key.ptr, pos.ptr, d_id, rstart.ptr, R, rcur.ptr, rinl.ptr, rkind.ptr,
           rflags.ptr, in_pos.ptr, me_pos.ptr, out.src.ptr, out.dst.ptr, out.val.ptr, out.flags.ptr, out.key.ptr, out.id.ptr,
           out.base.ptr);
    out.to_host(P);
}

void tensor_remove_plan(const EdgeTypeDev &type, const u64 *d_id, const u64 *d_src, const u64 *d_dst, u64 n, u64 nv, WritePlan &P) {
    const EType t = etype(type);
    const u32 grid = (u32)ctx().num_sms * 8;
    DevBuf<u64> key(n), id(n), rstart;
    // Compulsory bytes ("tensor_write"): 24 per batch edge (id, src, dst read once), 64 per distinct pair (the row pointers of dp,
    // dm, m and mt it probes; the merged id lists of multi-edge pairs are not counted), 25 per pair record and 17 per me entry.
    TimedScope ts(TK_TENSOR_WRITE, 0);
    LAUNCH(k_wp_keys, grid_for(n, 256, grid), 256, 0, d_src, d_dst, d_id, n, key.ptr, id.ptr);
    sort_pairs_u64(id.ptr, key.ptr, n, 60);                     // ids < 2^60, then a stable sort by pair: (key, id) ascending
    sort_pairs_u64(key.ptr, id.ptr, n, key_bits(nv));
    const u64 R = mark_runs(key.ptr, n, grid, rstart);
    DevBuf<u64> rval(R), pr_pos, me_pos;
    DevBuf<uint8_t> rflags(R);
    DevBuf<u32> pr_cnt(R + 1), me_cnt(R + 1);
    CUDA_TRY(cudaMemsetAsync(pr_cnt.ptr + R, 0, sizeof(u32), stream()));
    CUDA_TRY(cudaMemsetAsync(me_cnt.ptr + R, 0, sizeof(u32), stream()));
    LAUNCH(k_rm_count, grid_for(R, 256, grid), 256, 0, t, key.ptr, id.ptr, rstart.ptr, R, rval.ptr, rflags.ptr, pr_cnt.ptr, me_cnt.ptr);
    place(pr_cnt.ptr, me_cnt.ptr, R, pr_pos, me_pos, &P.nrec, &P.nme);
    ts.bytes = 24 * n + 64 * R + 25 * P.nrec + 17 * P.nme;
    PlanBufs out(P.nrec, P.nme);
    LAUNCH(k_rm_fill, grid_for(R, 256, grid), 256, 0, t, key.ptr, id.ptr, rstart.ptr, R, rval.ptr, rflags.ptr, pr_pos.ptr, me_pos.ptr,
           out.src.ptr, out.dst.ptr, out.val.ptr, out.flags.ptr, out.key.ptr, out.id.ptr, out.base.ptr);
    out.to_host(P);
}

} // namespace b200
