// graph_api.cu -- FalkorDB's batched relationship calls (include/b200grb.h): traversals, reachability, BFS and adjacency over
// relationship operands with pending writes, relationship ids, variable-length trails and Tensor write plans, each as one call.
// The entry points take their C linkage from b200grb.h; the handles and helpers they share with grb_api.cu are in handle.cuh.
#include "handle.cuh"

// ---- unions of relationship operands with pending writes: E = U_t (m[t] \ dm[t]) u dp[t], pattern only ----
// What the reference builds for a hop or a var-len walk over several relationship types (build_relationship_matrix_unrestricted,
// graph.rs:2520-2550: extract(T_1), then set_pattern(<!dm_t> m_t) and set_pattern(dp_t) per further type).  The union is exact:
// an entry that one type contributes survives another type's dm, and within a type dp wins over dm.  Walked by
// B200_reach_batch_delta and multiplied by the union hops of B200_Matrix_union_lmxm / B200_traverse_batch_union.
struct UnionOperand {
    GrB_Matrix m = nullptr, dp = nullptr, dm = nullptr;
    const DevCSR *ddp = nullptr;                 // dp's device form when it holds entries
    RepairPlan rp;                               // dm's repair plan (rp.ns == 0: nothing to repair)
    bool planned = false;                        // ddp and rp are set (union_plan)
};

static std::vector<UnionOperand> union_operands(const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops) {
    std::vector<UnionOperand> ops(nops);
    for (int t = 0; t < nops; t++) { ops[t].m = m[t]; ops[t].dp = dp ? dp[t] : nullptr; ops[t].dm = dm ? dm[t] : nullptr; }
    return ops;
}

// one lock over the operands' (m, dp, dm) and the extra handles
static MultiLock lock_all(const std::vector<UnionOperand> &ops, const std::vector<GrB_Matrix> &extra = {}) {
    uvec<GrB_Matrix> hs(extra.begin(), extra.end());
    for (const UnionOperand &o : ops) hs.insert(hs.end(), {o.m, o.dp, o.dm});
    return MultiLock(hs.begin(), hs.end());
}

// Y = F * E in frontier form (F at most 1024 rows), under the submission lock; *fl += sum_t flops(F * m[t]) + flops(F * dp[t]).
// The first operand with a repair plan goes first: it writes Y fresh and has the columns its dm touches recomputed in place
// (bits_repair overwrites columns, so it cannot accumulate).  Every further clean operand ORs into the same natural-order Y: the
// pushes skip zeroing Y and the pull ORs each row into the stored record.  A further operand with a repair plan (or every further
// operand with union_accum = 0) gets a bit-matrix of its own that is repaired, naturalised and ORed in.  pt_ok applies to a single
// operand only: the CSR push may then leave Y in the operand's hot-set order, as GrB_mxm does.
static void union_product(GrB_Matrix F, std::vector<UnionOperand> &ops, bool pt_ok, DevBits &Y, u64 *fl, int *path) {
    Context &cx = ctx();
    const size_t nops = ops.size();
    finish_pending(F);
    std::vector<UnionOperand *> order;
    for (UnionOperand &o : ops) if (o.rp.ns) { order.push_back(&o); break; }
    for (UnionOperand &o : ops) if (order.empty() || &o != order[0]) order.push_back(&o);
    DevBits Xcsr;
    for (size_t i = 0; i < nops; i++) {
        UnionOperand &o = *order[i];
        const bool own = i > 0 && (o.rp.ns || !cx.opt_union_accum);
        DevBits Z;
        DevBits &T = own ? Z : Y;
        u64 f = 0;
        const bool from_csr = frontier_product(F, o.m, nops == 1 && pt_ok, T, &f, path, i > 0 && !own);
        if (o.rp.ns) {
            // the repair gathers from F in bit form: a frontier still in CSR form is converted for it
            if (from_csr && !Xcsr.valid()) bits_from_csr(F->dev, Xcsr);
            ensure_devT(o.m);
            bits_repair(from_csr ? Xcsr : F->bits, o.m->devT, o.rp, T);
        }
        if (o.ddp) f += bits_apply_deltas(from_csr ? nullptr : &F->bits, from_csr ? &F->dev : nullptr, nullptr, o.ddp, T);
        *fl += f;
        if (own) { bits_naturalise(Z); bits_or(Y, Z); }
    }
}

// *U = a new BOOL matrix holding the union over the operands of their induced effective layers ((m \ dm) u dp restricted to the
// kept vertices and renumbered by rank, adj.cu), and with symmetric its union with its transpose.  keep null: vertices below n_out,
// U is n_out x n_out; else the strictly ascending keep[0 .. nkeep), U is nkeep x nkeep.  Arguments checked by the caller.
static GrB_Info effective_adjacency(GrB_Matrix *U, const std::vector<UnionOperand> &ops, u64 n_out, const GrB_Index *keep, u64 nkeep,
                                    bool symmetric) {
    const u64 rows = keep ? nkeep : n_out;
    GrB_Info info = GrB_Matrix_new(U, GrB_BOOL, rows, rows);
    if (info) return info;
    info = guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(ops, {*U});
        ensure_init();
        DevBuf<u64> dkeep;
        DevBuf<u32> rank;
        if (keep) {
            dkeep.alloc(nkeep ? nkeep : 1);
            h2d(dkeep.ptr, (const u64 *)keep, nkeep);
            adj_rank_table(dkeep.ptr, nkeep, ops[0].m->ncols, rank);
        }
        DevCSR S;
        bool have = false;
        for (const UnionOperand &o : ops) {
            ensure_dev(o.m);
            const DevCSR *ddm = nullptr;
            if (o.dm) { ensure_dev(o.dm); if (o.dm->dev.nnz) ddm = &o.dm->dev; }
            DevCSR E;
            adj_layer(o.m->dev, ddm, n_out, keep ? dkeep.ptr : nullptr, rank.ptr, nkeep, E);
            if (o.dp) {
                ensure_dev(o.dp);
                if (o.dp->dev.nnz) {                 // dp's layer is merged in whole: within a type dp wins over dm
                    DevCSR D, T;
                    adj_layer(o.dp->dev, nullptr, n_out, keep ? dkeep.ptr : nullptr, rank.ptr, nkeep, D);
                    ewise_union(E, D, false, T);
                    E = std::move(T);
                }
            }
            if (!have) { S = std::move(E); have = true; }
            else { DevCSR T; ewise_union(S, E, false, T); S = std::move(T); }
        }
        if (symmetric) {
            DevCSR ST, T;
            transpose_csr(S, ST, false);
            ewise_union(S, ST, false, T);
            S = std::move(T);
        }
        set_dev(*U, std::move(S));
        return GrB_SUCCESS;
    });
    if (info) GrB_Matrix_free(U);
    return info;
}

// U = the union of every operand's effective pattern (m \ dm) u dp over all n vertices
static GrB_Info reach_materialise(GrB_Matrix *U, std::vector<UnionOperand> &ops, u64 n) {
    return effective_adjacency(U, ops, n, nullptr, 0, false);
}

// per call, for the frontier form: deltas' pending tuples finished, dp's device form, and dm's repair plan (dm' and the repaired
// segments of m', the base's mirror built at commit)
static GrB_Info union_plan(std::vector<UnionOperand> &ops) {
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(ops);
        ensure_init();
        for (UnionOperand &o : ops) {
            o.planned = true;
            if (o.dp) { ensure_dev(o.dp); if (o.dp->dev.nnz) o.ddp = &o.dp->dev; }
            if (!o.dm) continue;
            ensure_dev(o.dm);
            if (!o.dm->dev.nnz) continue;
            ensure_devT(o.m);
            bits_repair_plan(o.dm->dev, o.m->devT, o.rp);
        }
        return GrB_SUCCESS;
    });
}

// the plans' device buffers go back to the pool
static void union_release(std::vector<UnionOperand> &ops) { guarded([&]() { GpuLock g; ops.clear(); return GrB_SUCCESS; }); }

// ---- union hops: F <- F * E, exact (no delta_lmxm over-masking) ----
// A union hop is prepared once per call: with F in frontier form (a BOOL F of at most 1024 rows and bits_mode != 0) the operands'
// repair plans, otherwise the union materialised once (reach_materialise) for the general GrB_mxm -- the reference's cost, paid
// per call rather than per hop.  last_flops of a union hop = sum_t flops(F * m[t]) + flops(F * dp[t]) on either path: the work
// the frontier form does, independent of how the operands overlap.
struct UnionHop {
    std::vector<UnionOperand> ops;
    GrB_Matrix U = nullptr;                      // the materialised union (row-wise path)
};

static bool union_frontier(u64 rows, u64 n) {
    return ctx().opt_bits_mode != 0 && bits_words_for(rows) != 0 && n < ((u64)1 << 32);
}

static GrB_Info union_hop_prepare(UnionHop &uh, bool frontier, u64 n) {
    return frontier ? union_plan(uh.ops) : reach_materialise(&uh.U, uh.ops, n);
}

static void union_hop_release(UnionHop &uh) {
    GrB_Matrix_free(&uh.U);
    union_release(uh.ops);
}

static GrB_Info union_hop_apply(GrB_Matrix F, UnionHop &uh) {
    if (uh.U) {
        u64 fl = 0;
        GrB_Info info = guarded([&]() {
            GpuLock g;
            MultiLock lk = lock_all(uh.ops, {F});
            ensure_init();
            ensure_dev(F);
            for (UnionOperand &o : uh.ops) {
                ensure_dev(o.m);
                fl += spgemm_flops(F->dev, o.m->dev);
                if (o.dp) { ensure_dev(o.dp); fl += spgemm_flops(F->dev, o.dp->dev); }
            }
            return GrB_SUCCESS;
        });
        if (!info) info = GrB_mxm(F, nullptr, nullptr, GxB_ANY_PAIR_BOOL, F, uh.U, nullptr);
        if (!info) { Context &cx = ctx(); cx.total_flops -= cx.last_flops.load(); cx.total_flops += fl; cx.last_flops = fl; }
        return info;
    }
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(uh.ops, {F});
        ensure_init();
        Context &cx = ctx();
        DevBits Y;
        u64 fl = 0;
        int path = 0;
        union_product(F, uh.ops, true, Y, &fl, &path);
        cx.last_flops = fl; cx.total_flops += fl; cx.last_path = (u64)path;
        set_bits(F, std::move(Y));
        if (cx.opt_sync_after_op) sync_stream();
        return GrB_SUCCESS;
    });
}

// nops >= 1 operands and their deltas: square, of one size, device-resident
static GrB_Info operands_check(const char *what, const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops) {
    CHECK_PTR(m);
    if (nops < 1) { tl_error = std::string(what) + ": nops < 1"; return GrB_INVALID_VALUE; }
    for (int t = 0; t < nops; t++) {
        CHECK_MAT(m[t]);
        if (dp && dp[t]) CHECK_MAT(dp[t]);
        if (dm && dm[t]) CHECK_MAT(dm[t]);
    }
    const u64 n = m[0]->nrows;
    for (int t = 0; t < nops; t++)
        for (GrB_Matrix X : {m[t], dp ? dp[t] : nullptr, dm ? dm[t] : nullptr})
            if (X && (X->nrows != n || X->ncols != n)) {
                tl_error = std::string(what) + ": operands and deltas must be square and equally sized"; return GrB_DIMENSION_MISMATCH;
            }
    for (int t = 0; t < nops; t++)
        for (GrB_Matrix X : {m[t], dp ? dp[t] : nullptr, dm ? dm[t] : nullptr})
            if (X && is_huge(X)) { tl_error = std::string(what) + ": host-resident operand"; return GrB_NOT_IMPLEMENTED; }
    return GrB_SUCCESS;
}

static GrB_Info device_ready() { return guarded([&]() { GpuLock g; ensure_init(); return GrB_SUCCESS; }); }

// The union hop as one call, the counterpart of B200_Matrix_delta_lmxm: F <- F * U_t (m[t] \ dm[t]) u dp[t].
GrB_Info B200_Matrix_union_lmxm(GrB_Matrix F, const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops) {
    CHECK_MAT(F);
    GrB_Info info = operands_check("union_lmxm", m, dp, dm, nops);
    if (info) return info;
    const u64 n = m[0]->nrows;
    if (F->ncols != n) { tl_error = "union_lmxm: F * m does not fit F"; return GrB_DIMENSION_MISMATCH; }
    if (is_huge(F)) { tl_error = "union_lmxm: host-resident frontier"; return GrB_NOT_IMPLEMENTED; }
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    UnionHop uh;
    uh.ops = union_operands(m, dp, dm, nops);
    info = union_hop_prepare(uh, F->type == T_BOOL && union_frontier(F->nrows, n), n);
    if (!info) info = union_hop_apply(F, uh);
    union_hop_release(uh);
    return info;
}

// ---- delta_lmxm as ONE C call (matrix.rs:1317-1402): F <- (F*m AND NOT F*dm) OR F*dp over GxB_ANY_PAIR_BOOL ----
// The reference composes three GrB_mxm calls and an eWiseAdd, each of which builds or rewrites a whole |F| x n bit-matrix.  In
// frontier form only the deltas' entries are touched here: F*m runs through GrB_mxm's frontier path unchanged, then the dm and dp
// terms are applied to the product in place (bits_apply_deltas) before it replaces F.  Where the frontier path does not apply
// (bits_mode 0, more than 1024 rows, or the automatic choice takes the general row-wise path) the three-call composition runs.
// last_flops = flops(F*m) + flops(F*dp) + flops(F*dm), as the composition reports them.
static GrB_Info delta_compose(GrB_Matrix F, GrB_Matrix m, GrB_Matrix dp, GrB_Matrix dm) {
    GrB_Index np = 0, nm = 0;
    GrB_Info info = GrB_SUCCESS;
    if (dp) info = GrB_Matrix_nvals(&np, dp);
    if (!info && dm) info = GrB_Matrix_nvals(&nm, dm);
    if (info) return info;
    if (!np && !nm) return GrB_mxm(F, nullptr, nullptr, GxB_ANY_PAIR_BOOL, F, m, nullptr);
    GrB_Matrix mk = nullptr, ac = nullptr;
    u64 flops = 0;
    auto product = [&](GrB_Matrix *out, GrB_Matrix D) {        // *out = F * D, dropped when empty
        GrB_Index nv = 0;
        GrB_Info e = GrB_Matrix_new(out, GrB_BOOL, F->nrows, m->ncols);
        if (!e) e = GrB_mxm(*out, nullptr, nullptr, GxB_ANY_PAIR_BOOL, F, D, nullptr);
        if (!e) { flops += ctx().last_flops.load(); e = GrB_Matrix_nvals(&nv, *out); }
        if (!e && !nv) GrB_Matrix_free(out);
        return e;
    };
    if (nm) info = product(&mk, dm);
    if (!info && np) info = product(&ac, dp);
    if (!info) info = GrB_mxm(F, mk, nullptr, GxB_ANY_PAIR_BOOL, F, m, mk ? GrB_DESC_RSC : nullptr);
    if (!info) flops += ctx().last_flops.load();
    if (!info && ac) info = GrB_Matrix_eWiseAdd_BinaryOp(F, nullptr, nullptr, GxB_ANY_BOOL, F, ac, nullptr);
    GrB_Matrix_free(&mk);
    GrB_Matrix_free(&ac);
    if (!info) ctx().last_flops = flops;
    return info;
}

GrB_Info B200_Matrix_delta_lmxm(GrB_Matrix F, GrB_Matrix m, GrB_Matrix dp, GrB_Matrix dm) {
    CHECK_MAT(F); CHECK_MAT(m);
    if (dp) CHECK_MAT(dp);
    if (dm) CHECK_MAT(dm);
    if (F->ncols != m->nrows || F->ncols != m->ncols) { tl_error = "delta_lmxm: F * m does not fit F"; return GrB_DIMENSION_MISMATCH; }
    for (GrB_Matrix D : {dp, dm})
        if (D && (D->nrows != m->nrows || D->ncols != m->ncols)) { tl_error = "delta_lmxm: delta dimensions differ from m"; return GrB_DIMENSION_MISMATCH; }
    if (!dp && !dm) return GrB_mxm(F, nullptr, nullptr, GxB_ANY_PAIR_BOOL, F, m, nullptr);
    bool done = false;
    GrB_Info info = guarded([&]() {
        GpuLock g;
        MultiLock lk{F, m, dp, dm};
        for (GrB_Matrix X : {F, m, dp, dm})
            if (is_huge(X)) throw GrbError(GrB_NOT_IMPLEMENTED, "delta_lmxm: host-resident matrix");
        ensure_init();
        const DevCSR *ddm = nullptr, *ddp = nullptr;
        if (dm) { ensure_dev(dm); if (dm->dev.nnz) ddm = &dm->dev; }      // pending tuples finish first (dm.wait())
        if (dp) { ensure_dev(dp); if (dp->dev.nnz) ddp = &dp->dev; }
        done = frontier_mxm(F, nullptr, F, m, Desc(), false, ddm, ddp);
        return GrB_SUCCESS;
    });
    if (info || done) return info;
    return delta_compose(F, m, dp, dm);
}

// F(i, sources[i]) = 1 for i < n: the source rows a batched traversal or reach starts from
static GrB_Info seed_sources(GrB_Matrix F, const GrB_Index *sources, u64 n) {
    GrB_Scalar one = nullptr;
    GrB_Info info = GrB_Scalar_new(&one, GrB_BOOL);
    if (!info) info = GrB_Scalar_setElement_BOOL(one, true);
    uvec<u64> rows(n);
    for (u64 i = 0; i < n; i++) rows[i] = i;
    if (!info) info = GxB_Matrix_build_Scalar(F, rows.data(), sources, one, n);
    GrB_Scalar_free(&one);
    return info;
}

// ---- the coalesced traversal as ONE C call (SURVEY 8f-1: CondTraverseOp's batch coalescing, cond_traverse.rs:600-608, 1264-1285) ----
// F(i, sources[i]) = 1;  F <- F * hops[0] * ... * hops[nhops-1] over GxB_ANY_PAIR_BOOL;  result rows to HOST memory.
//   B200_OUT_BITMAP : out_bits[row * words_per_row + (col >> 6)], one bit per slot.  The batch is processed in 128-row slices and
//                     slice k's device-to-host copy (second stream) overlaps slice k+1's hops; page-locked out_bits makes the
//                     copies asynchronous.
//   B200_OUT_CSR    : out_p[nsrc + 1], out_j[<= out_j_capacity]; GrB_INSUFFICIENT_SPACE (with *nvals_out = entries needed) when the
//                     buffer is too small.
//   B200_OUT_AUTO   : bitmap when the result holds more than one entry per 32 slots (fewer bytes over PCIe), else CSR; the choice
//                     is reported in *format_out.  Needs both output buffers.
// Composed from the public entry points (each takes the submission lock for its own duration), so other threads' calls interleave.
// Operands are hop-major: hop h owns hop_nops[h] consecutive entries of hops / dp / dm (hop_nops NULL: one each).  A delta hop
// (hop_union NULL or hop_union[h] == 0, one operand k) is B200_Matrix_delta_lmxm(F, hops[k], dp[k], dm[k]); a union hop is
// B200_Matrix_union_lmxm over its operands, prepared once per call (union_hop_prepare).  dp / dm NULL (B200_traverse_batch) or
// holding NULL entries: clean operands.
static GrB_Info traverse_impl(const GrB_Index *sources, GrB_Index nsrc, const int *hop_nops, const int *hop_union,
                              const GrB_Matrix *hops, const GrB_Matrix *dp, const GrB_Matrix *dm, int nhops, int format,
                              uint64_t *out_bits, uint64_t words_per_row, uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity,
                              uint64_t *nvals_out, uint64_t *flops_out, int *format_out) {
    CHECK_PTR(hops);
    if (nsrc) CHECK_PTR(sources);
    if (nhops < 1) { tl_error = "traverse_batch: nhops < 1"; return GrB_INVALID_VALUE; }
    std::vector<int> first(nhops + 1, 0);        // hop h's operands: [first[h], first[h + 1]) (hop_nops checked by the caller)
    for (int h = 0; h < nhops; h++) first[h + 1] = first[h] + (hop_nops ? hop_nops[h] : 1);
    const int nopd = first[nhops];
    for (int k = 0; k < nopd; k++) {
        CHECK_MAT(hops[k]);
        if (dp && dp[k]) CHECK_MAT(dp[k]);
        if (dm && dm[k]) CHECK_MAT(dm[k]);
    }
    if (format != B200_OUT_BITMAP && format != B200_OUT_CSR && format != B200_OUT_AUTO) { tl_error = "traverse_batch: unknown format"; return GrB_INVALID_VALUE; }
    if ((format != B200_OUT_CSR && !out_bits) || (format != B200_OUT_BITMAP && (!out_p || (!out_j && out_j_capacity)))) {
        tl_error = "traverse_batch: output buffer missing for the requested format"; return GrB_NULL_POINTER;
    }
    const u64 inner = hops[0]->nrows, ncols = hops[nopd - 1]->ncols;
    const u64 wpr = (ncols + 63) / 64;
    if (format != B200_OUT_CSR && words_per_row != wpr) { tl_error = "traverse_batch: words_per_row must be ceil(ncols / 64)"; return GrB_DIMENSION_MISMATCH; }
    // GrB_mxm(C = F, A = F, B) needs C's dimensions to match the product: a chain over square n x n operands (what the reference
    // stores, graph.rs:1191, 1211) keeps them; rectangular chains are rejected up front
    for (int k = 0; k < nopd; k++) {
        if (hops[k]->nrows != inner || hops[k]->ncols != inner) { tl_error = "traverse_batch: operands must be square and equally sized"; return GrB_DIMENSION_MISMATCH; }
        for (GrB_Matrix D : {dp ? dp[k] : nullptr, dm ? dm[k] : nullptr})
            if (D && (D->nrows != inner || D->ncols != inner)) { tl_error = "traverse_batch: delta dimensions differ from the hop's"; return GrB_DIMENSION_MISMATCH; }
    }
    GrB_Info info = GrB_SUCCESS;
    // union hops: plans (frontier form, for the rows of one F: a 128-row slice or the whole batch) or the materialised union
    std::vector<UnionHop> uhops(hop_union ? nhops : 0);
    const bool ufrontier = union_frontier(format == B200_OUT_BITMAP ? std::min<u64>(nsrc, 128) : nsrc, inner);
    for (int h = 0; h < (int)uhops.size() && !info; h++)
        if (hop_union[h]) {
            uhops[h].ops = union_operands(hops + first[h], dp ? dp + first[h] : nullptr, dm ? dm + first[h] : nullptr, first[h + 1] - first[h]);
            info = union_hop_prepare(uhops[h], ufrontier, inner);
        }
    u64 flops = 0, nvals = 0;
    int chosen = format;
    std::vector<B200_Ticket> tickets;
    auto run_hops = [&](GrB_Matrix F, u64 r0, u64 r1) -> GrB_Info {
        GrB_Info e = seed_sources(F, sources + r0, r1 - r0);
        for (int h = 0; h < nhops && !e; h++) {
            const int k = first[h];
            e = (hop_union && hop_union[h]) ? union_hop_apply(F, uhops[h])
                                            : B200_Matrix_delta_lmxm(F, hops[k], dp ? dp[k] : nullptr, dm ? dm[k] : nullptr);
            if (!e) flops += ctx().last_flops.load();
            if (!e && h + 1 < nhops && F->ncols != hops[first[h + 1]]->nrows) { tl_error = "traverse_batch: hop dimensions do not chain"; e = GrB_DIMENSION_MISMATCH; }
        }
        return e;
    };
    auto fresh = [&](GrB_Matrix *F, u64 rows) -> GrB_Info {
        // the frontier's column dimension follows the hops: n0 x n1 x ... (rectangular label ranges are n x n in the reference)
        return GrB_Matrix_new(F, GrB_BOOL, rows, inner);
    };
    if (!info && (format == B200_OUT_AUTO || format == B200_OUT_CSR)) {
        // density is known only after the hops: run the whole batch once, then pick the hand-off
        GrB_Matrix F = nullptr;
        info = fresh(&F, nsrc);
        if (!info) info = run_hops(F, 0, nsrc);
        if (!info) info = GrB_Matrix_nvals(&nvals, F);
        if (!info) {
            if (format == B200_OUT_AUTO) chosen = (nvals * 32 > nsrc * ncols) ? B200_OUT_BITMAP : B200_OUT_CSR;
            if (chosen == B200_OUT_BITMAP) info = B200_Matrix_export_bitmap(F, out_bits, wpr, nullptr, B200_LOC_HOST);
            else if (nvals > out_j_capacity) { tl_error = "traverse_batch: out_j too small"; info = GrB_INSUFFICIENT_SPACE; }
            else {
                info = GrB_Matrix_wait(F, GrB_MATERIALIZE);
                if (!info) info = B200_Matrix_export_CSR(F, out_p, out_j, nullptr, B200_LOC_HOST);
            }
        }
        GrB_Matrix_free(&F);
    } else if (!info) {
        const u64 per = 128;
        for (u64 r0 = 0; r0 < nsrc && !info; r0 += per) {
            const u64 r1 = std::min<u64>(nsrc, r0 + per);
            GrB_Matrix F = nullptr;
            info = fresh(&F, r1 - r0);
            if (!info) info = run_hops(F, r0, r1);
            B200_Ticket t = nullptr;
            if (!info) info = B200_Matrix_export_bitmap_async(F, out_bits + r0 * wpr, wpr, &t);
            if (!info) tickets.push_back(t);
            GrB_Matrix_free(&F);
        }
        for (B200_Ticket &t : tickets) { GrB_Info e = B200_Ticket_wait(&t); if (!info) info = e; }
        nvals = ~0ULL;       // not counted on this path (a popcount pass per slice would only serve this number)
    }
    for (UnionHop &uh : uhops) union_hop_release(uh);
    if (nvals_out) *nvals_out = nvals;
    if (flops_out) *flops_out = flops;
    if (format_out) *format_out = chosen;
    return info;
}

GrB_Info B200_traverse_batch(const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *hops, int nhops, int format,
                             uint64_t *out_bits, uint64_t words_per_row, uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity,
                             uint64_t *nvals_out, uint64_t *flops_out, int *format_out) {
    return traverse_impl(sources, nsrc, nullptr, nullptr, hops, nullptr, nullptr, nhops, format, out_bits, words_per_row, out_p, out_j,
                         out_j_capacity, nvals_out, flops_out, format_out);
}

// The same traversal over operands with pending writes: hop h is (m[h], dp[h], dm[h]) through B200_Matrix_delta_lmxm.
GrB_Info B200_traverse_batch_delta(const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *m, const GrB_Matrix *dp,
                                   const GrB_Matrix *dm, int nhops, int format, uint64_t *out_bits, uint64_t words_per_row,
                                   uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity, uint64_t *nvals_out, uint64_t *flops_out,
                                   int *format_out) {
    return traverse_impl(sources, nsrc, nullptr, nullptr, m, dp, dm, nhops, format, out_bits, words_per_row, out_p, out_j,
                         out_j_capacity, nvals_out, flops_out, format_out);
}

// The same traversal over hop groups: hop h is a delta hop (hop_union[h] == 0, hop_nops[h] == 1) or a union hop over its
// hop_nops[h] operands (B200_Matrix_union_lmxm).  Operands, validation and errors as B200_Matrix_union_lmxm.
GrB_Info B200_traverse_batch_union(const GrB_Index *sources, GrB_Index nsrc, const int *hop_nops, const int *hop_union, int nhops,
                                   const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int format, uint64_t *out_bits,
                                   uint64_t words_per_row, uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity,
                                   uint64_t *nvals_out, uint64_t *flops_out, int *format_out) {
    CHECK_PTR(hop_nops); CHECK_PTR(hop_union);
    if (nsrc) CHECK_PTR(sources);
    if (nhops < 1) { tl_error = "traverse_batch: nhops < 1"; return GrB_INVALID_VALUE; }
    int nopd = 0;
    for (int h = 0; h < nhops; h++) {
        if (hop_nops[h] < 1) { tl_error = "traverse_batch: a hop has no operand"; return GrB_INVALID_VALUE; }
        if (hop_nops[h] > 1 && !hop_union[h]) { tl_error = "traverse_batch: a delta hop takes one operand"; return GrB_INVALID_VALUE; }
        nopd += hop_nops[h];
    }
    GrB_Info info = operands_check("traverse_batch_union", m, dp, dm, nopd);
    if (!info) info = device_ready();           // no device: fail before any host work
    if (info) return info;
    return traverse_impl(sources, nsrc, hop_nops, hop_union, m, dp, dm, nhops, format, out_bits, words_per_row, out_p, out_j,
                         out_j_capacity, nvals_out, flops_out, format_out);
}

// ---- multi-source reachability as ONE C call (SURVEY 8f-1: the multiplicity-insensitive core of CondVarLenTraverse with
// emit_path = false, cond_var_len_traverse.rs:196, and of AllShortestPaths' BFS phase, all_shortest_paths.rs:7-25) ----
// Row i of *reached = every vertex reachable from sources[i] by a walk of 1..max_hops edges of A (max_hops < 0: until no row finds
// a new vertex); with include_sources the zero-length walk (i, sources[i]) belongs to the result and is never re-discovered.
// Each level is F<!R, replace, struct> = F*A (GrB_DESC_RSC, matrix.rs:1386) followed by R = R u F (matrix.rs:1398-1400); both stay
// in device frontier form for <= 1024 sources.  Composed from the public entry points.  *reached is a new nsrc x n BOOL matrix.
//
// B200_reach_batch_delta walks A = U_t (m[t] \ dm[t]) u dp[t] exactly (no delta_lmxm over-masking).  One operand without deltas
// (B200_reach_batch) issues the calls above unchanged.  Otherwise a level in frontier form is reach_hop: Y = F * A through
// union_product (per operand Y = F*m[t] through the usual dispatch, the columns dm[t] touches recomputed from m[t]'s transpose
// mirror without the deleted in-edges (bits_repair), then the dp[t] term, the operands' products ORed into one Y), and only then is
// the reached set masked out, so a dp edge cannot re-add a vertex already reached.  With bits_mode -1 the dirty reach stays in frontier form whenever it is legal (a tiny
// hop-1 frontier takes the CSR push there): the row-wise path would first need every dirty operand rewritten, O(nnz(m)) per call.
// Where the frontier path does not apply (bits_mode 0, more than 1024 sources) every dirty operand is materialised once per call
// by the adjacency builder (effective_adjacency, identity form) and the level runs the calls above over their union.

// One level in frontier form: F <- (F * A) AND NOT R (R only when masked).  F has at most 1024 rows.  Runs under the submission
// lock.  One operand and no mask: the CSR push may leave Y in the operand's hot-set order, as GrB_mxm does.
static void reach_hop(GrB_Matrix F, GrB_Matrix R, bool masked, std::vector<UnionOperand> &ops) {
    Context &cx = ctx();
    DevBits acc;
    u64 fl = 0;
    int path = 0;
    union_product(F, ops, !masked, acc, &fl, &path);
    if (masked) {
        bits_naturalise(acc);
        ensure_bits(R);
        bits_andnot(acc, R->bits);
    }
    cx.last_flops = fl; cx.total_flops += fl; cx.last_path = (u64)path;
    set_bits(F, std::move(acc));
    if (cx.opt_sync_after_op) sync_stream();
}

// planned (optional): on success, receives the operands' frontier-form plan when the reach built one (left empty otherwise), so a
// caller that runs further levels over the same operands need not plan them again; it releases them with union_release.
static GrB_Info reach_impl(GrB_Matrix *reached, const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *m, const GrB_Matrix *dp,
                           const GrB_Matrix *dm, int nops, int64_t max_hops, int include_sources, int64_t *levels_out,
                           std::vector<UnionOperand> *planned = nullptr) {
    const u64 n = m[0]->ncols;
    bool clean = nops == 1;
    for (int t = 0; t < nops && clean; t++)
        for (GrB_Matrix D : {dp ? dp[t] : nullptr, dm ? dm[t] : nullptr}) {
            GrB_Index nv = 0;
            if (!D) continue;
            GrB_Info e = GrB_Matrix_nvals(&nv, D);
            if (e) return e;
            if (nv) clean = false;
        }
    GrB_Matrix U = nullptr;                      // the materialised union, when a level runs the row-wise calls
    GrB_Info info = GrB_SUCCESS;
    std::vector<UnionOperand> ops = union_operands(m, dp, dm, nops);
    const bool frontier = ctx().opt_bits_mode != 0 && bits_words_for(nsrc) != 0;
    const bool U_built = !clean && !frontier;
    if (U_built) info = reach_materialise(&U, ops, n);
    else if (!clean) info = union_plan(ops);
    GrB_Matrix A = U ? U : m[0];                 // the operand of the row-wise calls
    GrB_Matrix F = nullptr, R = nullptr;
    if (!info) info = GrB_Matrix_new(&F, GrB_BOOL, nsrc, n);
    if (!info) info = GrB_Matrix_new(&R, GrB_BOOL, nsrc, n);
    if (!info && nsrc) info = seed_sources(F, sources, nsrc);
    if (!info && nsrc && include_sources) info = seed_sources(R, sources, nsrc);
    int64_t level = 0;
    while (!info && nsrc && (max_hops < 0 || level < max_hops)) {
        GrB_Index rn = 0, fn = 0;
        info = GrB_Matrix_nvals(&rn, R);
        if (info) break;
        if (!clean && !U) {
            info = guarded([&]() {
                GpuLock g;
                MultiLock lk = lock_all(ops, {F, R});
                ensure_init();
                reach_hop(F, R, rn != 0, ops);
                return GrB_SUCCESS;
            });
        } else {
            info = rn ? GrB_mxm(F, R, nullptr, GxB_ANY_PAIR_BOOL, F, A, GrB_DESC_RSC)
                      : GrB_mxm(F, nullptr, nullptr, GxB_ANY_PAIR_BOOL, F, A, nullptr);
        }
        if (!info) info = GrB_Matrix_nvals(&fn, F);
        if (info || fn == 0) break;
        info = GrB_Matrix_eWiseAdd_BinaryOp(R, nullptr, nullptr, GxB_ANY_BOOL, R, F, nullptr);
        level++;
    }
    GrB_Matrix_free(&F);
    GrB_Matrix_free(&U);
    if (!info && planned && !clean && !U_built) *planned = std::move(ops);
    else if (!clean) union_release(ops);
    if (info) { GrB_Matrix_free(&R); return info; }
    if (levels_out) *levels_out = level;
    *reached = R;
    return GrB_SUCCESS;
}

GrB_Info B200_reach_batch(GrB_Matrix *reached, const GrB_Index *sources, GrB_Index nsrc, GrB_Matrix A, int64_t max_hops,
                          int include_sources, int64_t *levels_out) {
    CHECK_PTR(reached); CHECK_MAT(A);
    if (nsrc) CHECK_PTR(sources);
    if (A->nrows != A->ncols) { tl_error = "reach_batch: A must be square"; return GrB_DIMENSION_MISMATCH; }
    return reach_impl(reached, sources, nsrc, &A, nullptr, nullptr, 1, max_hops, include_sources, levels_out);
}

GrB_Info B200_reach_batch_delta(GrB_Matrix *reached, const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *m,
                                const GrB_Matrix *dp, const GrB_Matrix *dm, int nops, int64_t max_hops, int include_sources,
                                int64_t *levels_out) {
    CHECK_PTR(reached);
    if (nsrc) CHECK_PTR(sources);
    GrB_Info info = operands_check("reach_batch_delta", m, dp, dm, nops);
    if (!info) info = device_ready();           // no device: fail before any host work
    if (info) return info;
    return reach_impl(reached, sources, nsrc, m, dp, dm, nops, max_hops, include_sources, levels_out);
}

// ---- single-source BFS over relationship operands with pending writes (algo.BFS, algo_procedures.rs:1021-1166) ----
// The reference builds A = U_t (m[t] \ dm[t]) u dp[t] afresh on every call (build_adjacency_matrix, graph.rs:3870-3893) and runs
// LAGr_BreadthFirstSearch_Extended on it.  Here the direction-optimising engine walks the operands in place: each base's transpose
// mirror and out-degree table are cached on its handle (ensure_devT, bfs_deg) and reused until the base changes; only the deltas'
// transposes are built per call.  One operand without deltas is exactly B200_Matrix_prepare(A, 1) + B200_bfs_ex.
GrB_Info B200_bfs_delta(const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops, GrB_Index src, int64_t max_level,
                        int64_t dest, int64_t *level, int64_t *parent, int location, B200_BfsInfo *info_out) {
    CHECK_PTR(level);
    GrB_Info info = operands_check("bfs_delta", m, dp, dm, nops);
    if (info) return info;
    const u64 n = m[0]->nrows;
    if (src >= n || (dest >= 0 && (u64)dest >= n)) { tl_error = "bfs_delta: src or dest out of range"; return GrB_INVALID_INDEX; }
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(union_operands(m, dp, dm, nops));
        ensure_init();
        // the deltas that hold entries, on the device
        std::vector<const DevCSR *> ddp(nops, nullptr), ddm(nops, nullptr);
        bool clean = nops == 1;
        for (int t = 0; t < nops; t++) {
            GrB_Matrix P = dp ? dp[t] : nullptr, M = dm ? dm[t] : nullptr;
            if (P && matrix_nvals(P)) { ensure_dev(P); ddp[t] = &P->dev; clean = false; }
            if (M && matrix_nvals(M)) { ensure_dev(M); ddm[t] = &M->dev; clean = false; }
        }
        if (clean) {
            ensure_devT(m[0]);
            bfs_staged(m[0], &m[0]->devT, n, 0, nullptr, src, max_level, dest, level, parent, location, info_out);
            return GrB_SUCCESS;
        }
        std::vector<DevCSR> dT(2 * nops);           // dp' and dm', built per call (the deltas change with every write)
        std::vector<BfsOperand> ops(nops);
        for (int t = 0; t < nops; t++) {
            GrB_Matrix A = m[t];
            ensure_devT(A);
            if (!A->bfs_deg_valid) { bfs_build_degrees(A->dev, n, 0, n, nullptr, A->bfs_deg, &A->bfs_edges); A->bfs_deg_valid = true; }
            if (ddp[t]) transpose_csr(*ddp[t], dT[2 * t], false);
            if (ddm[t]) transpose_csr(*ddm[t], dT[2 * t + 1], false);
            ops[t] = BfsOperand{&A->dev, &A->devT, ddp[t], ddp[t] ? &dT[2 * t] : nullptr, ddm[t], ddm[t] ? &dT[2 * t + 1] : nullptr,
                                A->bfs_deg.ptr, A->bfs_edges};
        }
        DevBuf<u32> deg;
        u64 total = 0;
        bfs_delta_degrees(ops, n, deg, &total);
        bfs_staged(m[0], nullptr, n, 0, nullptr, src, max_level, dest, level, parent, location, info_out, &ops, deg.ptr, total);
        return GrB_SUCCESS;
    });
}

// ---- the adjacency of algo.pageRank / algo.WCC / algo.labelPropagation over operands with pending writes ----
// The reference builds it afresh on every call: build_adjacency_matrix or build_symmetric_adjacency_matrix, then dup + resize to
// node_count + deleted_nodes_count (algo_procedures.rs:718-724, 816-822, 1207-1213), or, with a label filter, a host walk over every
// edge of every named tensor remapped through a hash map (build_compact_adj_*_from_tensors, :535-670).  Here both are one device
// call over the operands as they stand (effective_adjacency); only the kept rows of each layer are read.
GrB_Info B200_adjacency_delta(GrB_Matrix *A, const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops, GrB_Index n_out,
                              const GrB_Index *keep, GrB_Index nkeep, int symmetric) {
    CHECK_PTR(A);
    GrB_Info info = operands_check("adjacency_delta", m, dp, dm, nops);
    if (info) return info;
    const u64 n = m[0]->ncols;
    if (keep) {
        for (GrB_Index k = 0; k < nkeep; k++)
            if (keep[k] >= n || (k && keep[k] <= keep[k - 1])) {
                tl_error = "adjacency_delta: keep must be strictly ascending vertex ids below ncols(m)"; return GrB_INVALID_INDEX;
            }
    } else if (n_out >= ((u64)1 << 32)) {
        tl_error = "adjacency_delta: n_out must be below 2^32"; return GrB_INVALID_VALUE;
    }
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    std::vector<UnionOperand> ops = union_operands(m, dp, dm, nops);
    return effective_adjacency(A, ops, n_out, keep, keep ? nkeep : 0, symmetric != 0);
}

// ---- relationship ids of a batch of rows (expand_row / bind_edge / ExpandInto's Tensor::get, cond_traverse.rs:663-702, 844-935,
// expand_into.rs:121-258) in one call: edges.cu.  The me layers stay host-resident; their stores go to the device once per handle
// and change (GB_Matrix_opaque::ids, dropped by invalidate_aux).
static const DevIdStore *id_store(GrB_Matrix A) {
    if (!A) return nullptr;
    ensure_host(A);
    if (!A->ids.valid) {
        const HostStore &h = A->host;
        A->ids.upload(h.hrow.data(), h.hptr.data(), h.hcol.data(), h.hrow.size());
    }
    return &A->ids;
}

static const DevCSR *dev_or_null(GrB_Matrix X) {
    if (!X) return nullptr;
    ensure_dev(X);
    return &X->dev;
}

// every type's nine layers: valid handles (mt present when need_mt), UINT64 forward layers m / dp, the forward and transpose
// layers square and of one size, device-resident
static GrB_Info layers_check(const char *what, const B200_TensorLayers *types, int ntypes, bool need_mt) {
    for (int t = 0; t < ntypes; t++) {
        const B200_TensorLayers &L = types[t];
        CHECK_MAT(L.m);
        for (GrB_Matrix X : {L.dp, L.dm, L.mt, L.mt_dp, L.mt_dm, L.me, L.me_dp, L.me_dm}) if (X) CHECK_MAT(X);
        if (need_mt && !L.mt) { tl_error = std::string(what) + ": the transpose mt is missing"; return GrB_NULL_POINTER; }
        if (L.m->type != T_UINT64 || (L.dp && L.dp->type != T_UINT64)) {
            tl_error = std::string(what) + ": the forward layers m / dp must be UINT64 (edge ids)"; return GrB_DOMAIN_MISMATCH;
        }
    }
    const u64 nv = types[0].m->nrows;
    for (int t = 0; t < ntypes; t++) {
        const B200_TensorLayers &L = types[t];
        for (GrB_Matrix X : {L.m, L.dp, L.dm, L.mt, L.mt_dp, L.mt_dm})
            if (X && (X->nrows != nv || X->ncols != nv)) {
                tl_error = std::string(what) + ": forward and transpose layers must be square and equally sized"; return GrB_DIMENSION_MISMATCH;
            }
    }
    if (is_huge(types[0].m)) { tl_error = std::string(what) + ": host-resident forward or transpose layers"; return GrB_NOT_IMPLEMENTED; }
    return GrB_SUCCESS;
}

// one lock over every type's nine layers and the extra handles
static MultiLock lock_all(const B200_TensorLayers *types, int ntypes, const std::vector<GrB_Matrix> &extra = {}) {
    uvec<GrB_Matrix> hs(extra.begin(), extra.end());
    for (int t = 0; t < ntypes; t++) {
        const B200_TensorLayers &L = types[t];
        hs.insert(hs.end(), {L.m, L.dp, L.dm, L.mt, L.mt_dp, L.mt_dm, L.me, L.me_dp, L.me_dm});
    }
    return MultiLock(hs.begin(), hs.end());
}

// every type's layers as edges.cu and trails.cu read them: the transpose's only for incoming edges
static std::vector<EdgeTypeDev> edge_types_dev(const B200_TensorLayers *types, int ntypes, int dir) {
    std::vector<EdgeTypeDev> td(ntypes);
    const bool rev = dir != B200_DIR_OUT;
    for (int t = 0; t < ntypes; t++) {
        const B200_TensorLayers &L = types[t];
        td[t] = EdgeTypeDev{dev_or_null(L.m), dev_or_null(L.dp), dev_or_null(L.dm), rev ? dev_or_null(L.mt) : nullptr,
                            rev ? dev_or_null(L.mt_dp) : nullptr, rev ? dev_or_null(L.mt_dm) : nullptr, id_store(L.me),
                            id_store(L.me_dp), id_store(L.me_dm)};
    }
    return td;
}

GrB_Info B200_expand_edges(const GrB_Index *sources, const GrB_Index *targets, GrB_Index n, const B200_TensorLayers *types,
                           int ntypes, int dir, int mode, uint64_t *out_p, uint32_t *out_node, uint64_t *out_edge,
                           uint16_t *out_type, uint8_t *out_rev, uint64_t out_capacity, uint64_t *nout) {
    CHECK_PTR(types); CHECK_PTR(out_p); CHECK_PTR(nout);
    if (n) CHECK_PTR(sources);
    if (out_capacity) { CHECK_PTR(out_node); CHECK_PTR(out_edge); }
    if (ntypes < 1 || ntypes > 65536 || dir < B200_DIR_OUT || dir > B200_DIR_BOTH || mode < B200_EDGES_ALL || mode > B200_EDGES_FIRST) {
        tl_error = "expand_edges: ntypes outside 1 .. 65536 (out_type is 16 bits), or dir / mode out of range"; return GrB_INVALID_VALUE;
    }
    GrB_Info info = layers_check("expand_edges", types, ntypes, dir != B200_DIR_OUT);
    if (info) return info;
    const u64 nv = types[0].m->nrows;
    for (u64 i = 0; i < n; i++)
        if (sources[i] >= nv || (targets && targets[i] >= nv)) { tl_error = "expand_edges: vertex id out of range"; return GrB_INVALID_INDEX; }
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(types, ntypes);
        ensure_init();
        const std::vector<EdgeTypeDev> td = edge_types_dev(types, ntypes, dir);
        DevBuf<u64> ds(n), dtg(targets ? n : 0);
        h2d(ds.ptr, (const u64 *)sources, n);
        if (targets) h2d(dtg.ptr, (const u64 *)targets, n);
        const u64 total = edge_expand(ds.ptr, targets ? dtg.ptr : nullptr, n, td, dir, mode, out_p, out_node, out_edge, out_type,
                                      out_rev, out_capacity);
        *nout = total;
        if (total > out_capacity) { tl_error = "expand_edges: output capacity too small (*nout = entries needed)"; return GrB_INSUFFICIENT_SPACE; }
        return GrB_SUCCESS;
    });
}

// ---- CondVarLenTraverse's trails (cond_var_len_traverse.rs:152-386) for a batch of starts in one call: trails.cu.  The type
// layers are read as B200_expand_edges reads them; the destination labels' (m, dp, dm) become one bitmap on the device.
GrB_Info B200_var_len_trails(const GrB_Index *starts, const int64_t *dests, GrB_Index nstarts, const B200_TensorLayers *types,
                             int ntypes, int dir, uint64_t min_hops, uint64_t max_hops, const GrB_Matrix *lab_m,
                             const GrB_Matrix *lab_dp, const GrB_Matrix *lab_dm, int nlabels, uint64_t tree_capacity,
                             uint64_t *out_p, uint32_t *out_end, uint32_t *out_hops, uint64_t out_capacity,
                             uint64_t *path_edge, uint32_t *path_node, uint64_t path_capacity, uint64_t *nout, uint64_t *npath) {
    CHECK_PTR(types); CHECK_PTR(out_p); CHECK_PTR(nout); CHECK_PTR(npath);
    if (nstarts) CHECK_PTR(starts);
    if (out_end) CHECK_PTR(out_hops);
    if (path_edge) CHECK_PTR(path_node);
    if (ntypes < 1 || ntypes > 65536 || dir < B200_DIR_OUT || dir > B200_DIR_BOTH || nlabels < 0) {
        tl_error = "var_len_trails: ntypes outside 1 .. 65536, dir out of range, or nlabels < 0"; return GrB_INVALID_VALUE;
    }
    if (nlabels) CHECK_PTR(lab_m);
    GrB_Info info = layers_check("var_len_trails", types, ntypes, dir != B200_DIR_OUT);
    if (info) return info;
    const u64 nv = types[0].m->nrows;
    bool missing = false;
    std::vector<GrB_Matrix> labs;                // (m, dp, dm) per present label
    for (int k = 0; k < nlabels; k++) {
        GrB_Matrix m = lab_m[k], dp = lab_dp ? lab_dp[k] : nullptr, dm = lab_dm ? lab_dm[k] : nullptr;
        for (GrB_Matrix X : {m, dp, dm}) if (X) CHECK_MAT(X);
        if (!m) { missing = true; continue; }
        labs.insert(labs.end(), {m, dp, dm});
    }
    for (GrB_Matrix X : labs)
        if (X && (X->nrows != nv || X->ncols != nv)) {
            tl_error = "var_len_trails: label layers must be n x n"; return GrB_DIMENSION_MISMATCH;
        }
    for (GrB_Matrix X : labs)
        if (is_huge(X)) { tl_error = "var_len_trails: host-resident label layers"; return GrB_NOT_IMPLEMENTED; }
    for (u64 i = 0; i < nstarts; i++)
        if (starts[i] >= nv || (dests && dests[i] >= 0 && (u64)dests[i] >= nv)) {
            tl_error = "var_len_trails: start or destination out of range"; return GrB_INVALID_INDEX;
        }
    auto empty = [&]() {                         // no trail emits
        for (u64 i = 0; i <= nstarts; i++) out_p[i] = 0;
        *nout = 0; *npath = 0;
        return GrB_SUCCESS;
    };
    if (nstarts == 0 || min_hops > max_hops) return empty();
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(types, ntypes, labs);
        ensure_init();
        if (missing) return empty();             // a label the graph lacks: every trail is walked, none emits (:162, :316)
        const std::vector<EdgeTypeDev> td = edge_types_dev(types, ntypes, dir);
        std::vector<LabelDev> ld;
        for (size_t k = 0; k < labs.size(); k += 3)
            ld.push_back(LabelDev{dev_or_null(labs[k]), dev_or_null(labs[k + 1]), dev_or_null(labs[k + 2])});
        TrailsOut o{out_p, out_end, out_hops, path_edge, path_node, out_capacity, path_capacity};
        const int r = var_len_trails((const u64 *)starts, (const i64 *)dests, nstarts, td, dir, min_hops, max_hops, ld, nv, tree_capacity, o);
        if (r == 2) {
            *nout = *npath = UINT64_MAX;
            tl_error = "var_len_trails: the stored trail tree would exceed tree_capacity entries";
            return GrB_INSUFFICIENT_SPACE;
        }
        *nout = o.nout; *npath = o.npath;
        if (r == 1) { tl_error = "var_len_trails: output capacity too small (*nout / *npath = what is needed)"; return GrB_INSUFFICIENT_SPACE; }
        return GrB_SUCCESS;
    });
}

// ---- CondVarLenTraverse's DISTINCT endpoints of a bidirectional pattern (a)-[*min..max]-(b), min <= 1, for a batch of starts.
// Every v != s: B200_reach_batch_delta's walk over each type's forward and transpose layers (a shortest walk is a path, hence a
// trail); the start itself: a cycle through it of at most max_hops edges (var_len_reach.cu), whose longer cases run masked
// levels of reach_hop over the same operands in closure rows of at most 1024.
// ops: the reach's operands, planned by it (reach_impl's `planned`) or, when the reach materialised their union, not yet planned
static GrB_Info reach_both_closure(GrB_Matrix R, const GrB_Index *starts, GrB_Index nstarts, const B200_TensorLayers *types,
                                   int ntypes, std::vector<UnionOperand> &ops, uint64_t max_hops) {
    const u64 n = types[0].m->nrows;
    VlbPlan P;
    GrB_Info info = guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(types, ntypes);
        ensure_init();
        vlb_plan((const u64 *)starts, nstarts, edge_types_dev(types, ntypes, B200_DIR_BOTH), max_hops, P);
        return GrB_SUCCESS;
    });
    if (!info && P.rows && !ops.front().planned) info = union_plan(ops);
    for (u64 r0 = 0; r0 < P.rows && !info; r0 += 1024) {
        const u64 r1 = std::min<u64>(P.rows, r0 + 1024);
        GrB_Matrix F = nullptr, V = nullptr;
        info = GrB_Matrix_new(&F, GrB_BOOL, r1 - r0, n);
        if (!info) info = GrB_Matrix_new(&V, GrB_BOOL, r1 - r0, n);
        if (!info) info = guarded([&]() {
            GpuLock g;
            MultiLock lk = lock_all(ops, {F, V});
            DevBits fb, vb;
            vlb_seed(P, r0, r1, n, fb, vb);
            set_bits(F, std::move(fb));
            set_bits(V, std::move(vb));
            // the middle of a cycle of g <= max_hops edges is a path of g - 2 edges
            for (u64 level = 0; level + 2 < max_hops; level++) {
                reach_hop(F, V, true, ops);
                if (!vlb_level(P, r0, r1, F->bits)) break;
                bits_or(V->bits, F->bits);
            }
            return GrB_SUCCESS;
        });
        GrB_Matrix_free(&F);
        GrB_Matrix_free(&V);
    }
    union_release(ops);
    if (!info) info = guarded([&]() {
        GpuLock g;
        MultiLock lk{R};
        if (R->bits_valid) {
            ensure_bits(R);
            DevBits b = std::move(R->bits);
            vlb_fix_bits(P, b);
            set_bits(R, std::move(b));
        } else {
            ensure_dev(R);
            DevCSR out;
            vlb_fix_csr(P, R->dev, out);
            set_dev(R, std::move(out));
        }
        return GrB_SUCCESS;
    });
    guarded([&]() { GpuLock g; P = VlbPlan(); return GrB_SUCCESS; });   // the plan's buffers go back to the pool
    return info;
}

GrB_Info B200_var_len_reach_both(GrB_Matrix *reached, const GrB_Index *starts, GrB_Index nstarts, const B200_TensorLayers *types,
                                 int ntypes, uint64_t min_hops, uint64_t max_hops) {
    CHECK_PTR(reached); CHECK_PTR(types);
    if (nstarts) CHECK_PTR(starts);
    if (ntypes < 1 || ntypes > 65536) { tl_error = "var_len_reach_both: ntypes outside 1 .. 65536"; return GrB_INVALID_VALUE; }
    GrB_Info info = layers_check("var_len_reach_both", types, ntypes, true);
    if (info) return info;
    const u64 nv = types[0].m->nrows;
    for (u64 i = 0; i < nstarts; i++)
        if (starts[i] >= nv) { tl_error = "var_len_reach_both: start out of range"; return GrB_INVALID_INDEX; }
    if (min_hops > 1) { tl_error = "var_len_reach_both: min_hops > 1 is not a reach (a walk is not a trail)"; return GrB_NOT_IMPLEMENTED; }
    if (nstarts == 0 || min_hops > max_hops) return GrB_Matrix_new(reached, GrB_BOOL, nstarts, nv);
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    std::vector<GrB_Matrix> m, dp, dm;           // each type's forward layers, then its transpose's: the pattern of G'
    for (int t = 0; t < ntypes; t++) {
        const B200_TensorLayers &L = types[t];
        m.insert(m.end(), {L.m, L.mt}); dp.insert(dp.end(), {L.dp, L.mt_dp}); dm.insert(dm.end(), {L.dm, L.mt_dm});
    }
    GrB_Matrix R = nullptr;
    std::vector<UnionOperand> ops;               // the reach's plan, reused by the closure's levels
    info = reach_impl(&R, starts, nstarts, m.data(), dp.data(), dm.data(), 2 * ntypes,
                      max_hops > (uint64_t)INT64_MAX ? -1 : (int64_t)max_hops, 1, nullptr, min_hops == 0 ? nullptr : &ops);
    if (info || min_hops == 0) { if (!info) *reached = R; return info; }
    if (ops.empty()) ops = union_operands(m.data(), dp.data(), dm.data(), 2 * ntypes);
    info = reach_both_closure(R, starts, nstarts, types, ntypes, ops, max_hops);
    if (info) { GrB_Matrix_free(&R); return info; }
    *reached = R;
    return GrB_SUCCESS;
}

// ---- allShortestPaths((a)-[:R*..max]->(b)) for a batch of bound pairs (AllShortestPathsOp::expand_row,
// all_shortest_paths.rs:82-302): all_shortest_paths.cu.  The type layers are read as B200_expand_edges reads them, the transpose
// of every type included: the paths are recovered from dst over incoming edges.
GrB_Info B200_all_shortest_paths(const GrB_Index *src, const GrB_Index *dst, GrB_Index npairs, const B200_TensorLayers *types,
                                 int ntypes, int dir, uint64_t max_hops, const uint64_t *first, uint64_t *out_count, uint32_t *out_len,
                                 uint64_t *out_p, uint64_t *path_edge, uint32_t *path_node, uint64_t edge_capacity, uint64_t *nedges) {
    CHECK_PTR(types); CHECK_PTR(out_p); CHECK_PTR(nedges);
    if (npairs) { CHECK_PTR(src); CHECK_PTR(dst); CHECK_PTR(out_count); CHECK_PTR(out_len); }
    if (path_edge) CHECK_PTR(path_node);
    if (ntypes < 1 || ntypes > 65536 || (dir != B200_DIR_OUT && dir != B200_DIR_BOTH)) {
        tl_error = "all_shortest_paths: ntypes outside 1 .. 65536, or dir not OUT / BOTH"; return GrB_INVALID_VALUE;
    }
    GrB_Info info = layers_check("all_shortest_paths", types, ntypes, true);
    if (info) return info;
    const u64 nv = types[0].m->nrows;
    for (u64 i = 0; i < npairs; i++)
        if (src[i] >= nv || dst[i] >= nv) { tl_error = "all_shortest_paths: src or dst out of range"; return GrB_INVALID_INDEX; }
    if (npairs == 0 || max_hops == 0) {          // no path: empty rows
        for (u64 i = 0; i < npairs; i++) { out_count[i] = 0; out_len[i] = 0; }
        for (u64 i = 0; i <= npairs; i++) out_p[i] = 0;
        *nedges = 0;
        return GrB_SUCCESS;
    }
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(types, ntypes);
        ensure_init();
        const u64 fl = all_shortest_paths((const u64 *)src, (const u64 *)dst, npairs, edge_types_dev(types, ntypes, B200_DIR_BOTH), dir,
                                          nv, max_hops, (u64)std::max<i64>(0, ctx().opt_shortest_path_budget), first, out_count,
                                          out_len, out_p, path_edge, path_node, edge_capacity, nedges);
        Context &cx = ctx();
        cx.last_flops = fl; cx.total_flops += fl;
        return GrB_SUCCESS;
    });
}

// ---- shortestPath((a)-[:R*min..max]->(b)) for a batch of bound pairs (ExprEval::eval_shortest_path, eval.rs:1296-1513) ----
// The reference runs a bidirectional BFS per row over versioned row iterators.  Here the pairs other than src == dst run together
// (shortest_path.cu): each side's neighbours are the union of its operands' effective rows, read from the layers as they stand.
GrB_Info B200_shortest_path(const GrB_Index *src, const GrB_Index *dst, GrB_Index npairs, const GrB_Matrix *fm, const GrB_Matrix *fdp,
                            const GrB_Matrix *fdm, int nf, const GrB_Matrix *bm, const GrB_Matrix *bdp, const GrB_Matrix *bdm, int nb,
                            uint64_t min_hops, uint64_t max_hops, uint64_t *out_p, uint32_t *path_node, uint64_t node_capacity,
                            uint64_t *nnodes) {
    CHECK_PTR(out_p); CHECK_PTR(nnodes);
    if (npairs) { CHECK_PTR(src); CHECK_PTR(dst); }
    if (node_capacity) CHECK_PTR(path_node);
    if (nf < 1 || nb < 1) { tl_error = "shortest_path: each side needs at least one operand"; return GrB_INVALID_VALUE; }
    if (min_hops > 1) { tl_error = "shortest_path: min_hops must be 0 or 1"; return GrB_INVALID_VALUE; }
    GrB_Info info = operands_check("shortest_path", fm, fdp, fdm, nf);
    if (!info) info = operands_check("shortest_path", bm, bdp, bdm, nb);
    if (info) return info;
    const u64 n = fm[0]->nrows;
    if (bm[0]->nrows != n) { tl_error = "shortest_path: operands and deltas must be square and equally sized"; return GrB_DIMENSION_MISMATCH; }
    for (u64 i = 0; i < npairs; i++)
        if (src[i] >= n || dst[i] >= n) { tl_error = "shortest_path: src or dst out of range"; return GrB_INVALID_INDEX; }
    if (npairs == 0) { out_p[0] = 0; *nnodes = 0; return GrB_SUCCESS; }
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    std::vector<u64> ps, pd, pos;                // the pairs the BFS runs for, and their rows
    for (u64 i = 0; i < npairs; i++)
        if (src[i] != dst[i]) { ps.push_back(src[i]); pd.push_back(dst[i]); pos.push_back(i); }
    std::vector<u64> len;
    std::vector<u32> nodes;
    info = guarded([&]() {
        GpuLock g;
        std::vector<UnionOperand> all = union_operands(fm, fdp, fdm, nf), b = union_operands(bm, bdp, bdm, nb);
        all.insert(all.end(), std::make_move_iterator(b.begin()), std::make_move_iterator(b.end()));
        MultiLock lk = lock_all(all);
        ensure_init();
        std::vector<SpOperand> sides[2];
        for (int k = 0; k < nf + nb; k++)
            sides[k >= nf].push_back(SpOperand{dev_or_null(all[k].m), dev_or_null(all[k].dp), dev_or_null(all[k].dm)});
        const u64 fl = ps.empty() ? 0 : shortest_path(ps.data(), pd.data(), ps.size(), sides[0], sides[1], n, max_hops,
                                                     (u64)std::max<i64>(0, ctx().opt_shortest_path_budget), len, nodes);
        Context &cx = ctx();
        cx.last_flops = fl; cx.total_flops += fl;
        return GrB_SUCCESS;
    });
    if (info) return info;
    // rows in input order: src == dst is the one-node path with min_hops == 0 and Null otherwise (eval.rs:1329, 1406)
    std::vector<u64> first(ps.size() + 1, 0);
    for (size_t k = 0; k < ps.size(); k++) first[k + 1] = first[k] + len[k];
    u64 total = 0;
    for (u64 i = 0, k = 0; i < npairs; i++) {
        out_p[i] = total;
        if (k < pos.size() && pos[k] == i) total += len[k++];
        else total += min_hops == 0 ? 1 : 0;
    }
    out_p[npairs] = total;
    *nnodes = total;
    if (total > node_capacity) { tl_error = "shortest_path: node_capacity too small (*nnodes = nodes needed)"; return GrB_INSUFFICIENT_SPACE; }
    for (u64 i = 0, k = 0; i < npairs; i++) {
        if (k < pos.size() && pos[k] == i) {
            std::copy(nodes.begin() + first[k], nodes.begin() + first[k + 1], path_node + out_p[i]);
            k++;
        } else if (min_hops == 0) {
            path_node[out_p[i]] = (uint32_t)src[i];
        }
    }
    return GrB_SUCCESS;
}

// ---- the read phase of a Tensor's relationship inserts and deletes (set_all_from_slices / remove_all, tensor.rs:333-629) for a
// whole batch in one call: writes.cu.  Only reads the layers; their pending tuples are finished like any device read's.
static_assert(B200_PLAN_COMMITTED == WP_COMMITTED && B200_PLAN_CANCEL == WP_CANCEL && B200_PLAN_MT_BASE == WP_MT_BASE &&
              B200_PLAN_EMPTIED == WP_EMPTIED && B200_PLAN_DEMOTED == WP_DEMOTED && B200_PLAN_M_HAS == WP_M_HAS &&
              B200_PLAN_M_EQ == WP_M_EQ, "plan flags");

static GrB_Info write_plan(const char *what, bool insert, const B200_TensorLayers *t, const GrB_Index *a, const GrB_Index *b,
                           const GrB_Index *c, GrB_Index n, uint64_t *rec_src, uint64_t *rec_dst, uint64_t *rec_val,
                           uint8_t *rec_flags, uint64_t *nrec, uint64_t *me_key, uint64_t *me_id, uint8_t *me_base, uint64_t *nme) {
    CHECK_PTR(t); CHECK_PTR(nrec); CHECK_PTR(nme);
    if (n) {
        CHECK_PTR(a); CHECK_PTR(b); CHECK_PTR(c);
        CHECK_PTR(rec_src); CHECK_PTR(rec_dst); CHECK_PTR(rec_val); CHECK_PTR(rec_flags);
        CHECK_PTR(me_key); CHECK_PTR(me_id); CHECK_PTR(me_base);
    }
    GrB_Info info = layers_check(what, t, 1, true);
    if (info) return info;
    const u64 nv = t->m->nrows;
    // insert: (a, b, c) = (srcs, dsts, ids); remove: (ids, srcs, dsts)
    const GrB_Index *src = insert ? a : b, *dst = insert ? b : c, *ids = insert ? c : a;
    for (u64 k = 0; k < n; k++)
        if (src[k] >= nv || dst[k] >= nv || ids[k] >= ((u64)1 << 60)) {
            tl_error = std::string(what) + ": a vertex id >= n or an edge id >= 2^60"; return GrB_INVALID_INDEX;
        }
    *nrec = 0; *nme = 0;
    if (n == 0) return GrB_SUCCESS;
    info = device_ready();                       // no device: fail before any host work
    if (info) return info;
    return guarded([&]() {
        GpuLock g;
        MultiLock lk = lock_all(t, 1);
        ensure_init();
        const EdgeTypeDev td{dev_or_null(t->m), dev_or_null(t->dp), dev_or_null(t->dm), dev_or_null(t->mt), nullptr, nullptr,
                             id_store(t->me), insert ? nullptr : id_store(t->me_dp), insert ? nullptr : id_store(t->me_dm)};
        DevBuf<u64> ds(n), dd(n), di(n);
        h2d(ds.ptr, (const u64 *)src, n);
        h2d(dd.ptr, (const u64 *)dst, n);
        h2d(di.ptr, (const u64 *)ids, n);
        WritePlan P{rec_src, rec_dst, rec_val, rec_flags, 0, me_key, me_id, me_base, 0};
        if (insert) tensor_insert_plan(td, ds.ptr, dd.ptr, di.ptr, n, nv, P);
        else tensor_remove_plan(td, di.ptr, ds.ptr, dd.ptr, n, nv, P);
        *nrec = P.nrec; *nme = P.nme;
        return GrB_SUCCESS;
    });
}

GrB_Info B200_Tensor_insert_plan(const B200_TensorLayers *t, const GrB_Index *srcs, const GrB_Index *dsts, const GrB_Index *ids,
                                 GrB_Index n, uint64_t *in_src, uint64_t *in_dst, uint64_t *in_val, uint8_t *in_flags, uint64_t *nin,
                                 uint64_t *me_key, uint64_t *me_id, uint8_t *me_base, uint64_t *nme) {
    return write_plan("insert_plan", true, t, srcs, dsts, ids, n, in_src, in_dst, in_val, in_flags, nin, me_key, me_id, me_base, nme);
}
GrB_Info B200_Tensor_remove_plan(const B200_TensorLayers *t, const GrB_Index *ids, const GrB_Index *srcs, const GrB_Index *dsts,
                                 GrB_Index n, uint64_t *pr_src, uint64_t *pr_dst, uint64_t *pr_val, uint8_t *pr_flags, uint64_t *npr,
                                 uint64_t *me_key, uint64_t *me_id, uint8_t *me_base, uint64_t *nme) {
    return write_plan("remove_plan", false, t, ids, srcs, dsts, n, pr_src, pr_dst, pr_val, pr_flags, npr, me_key, me_id, me_base, nme);
}
