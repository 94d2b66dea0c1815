"""Host-side mirror of the reference's GraphBLAS wrapper, method for method:
``Matrix<T>`` in graph/src/graph/graphblas/matrix.rs (new :1119/:1214, build :1186/:1281, set/get
:1143-1172/:1248-1275, lmxm/rmxm :930-968, delta_lmxm :1317-1402, element_wise_add :852, element_wise_multiply
:876, set_pattern :906, transpose :633, remove_all/select :824-845, wait :781, dup :1062, grown :700, iter :1471).
Everything is a direct call into libb200grb.so through the GraphBLAS C ABI (include/b200grb.h)."""
import ctypes as C
import enum

import numpy as np

from ._lib import lib, obj, check, GrbError, P, U64, I64, BfsInfo

GxB_SPARSITY_STATUS, GxB_SPARSITY_CONTROL, GxB_HYPER_HASH, GxB_WILL_WAIT = 7034, 7036, 7048, 7076
GrB_STORAGE_ORIENTATION_HINT = 100
GxB_HYPERSPARSE, GxB_SPARSE = 1, 2
GrB_MATERIALIZE = 1
U64_MAX = (1 << 64) - 1


class Descriptor(enum.Enum):
    """matrix.rs:223-255"""
    T0 = "T0"; T1 = "T1"; T0T1 = "T0T1"; C = "C"; CT0 = "CT0"; CT1 = "CT1"; CT0T1 = "CT0T1"
    S = "S"; ST0 = "ST0"; ST1 = "ST1"; ST0T1 = "ST0T1"; SC = "SC"; SCT0 = "SCT0"; SCT1 = "SCT1"; SCT0T1 = "SCT0T1"
    R = "R"; RT0 = "RT0"; RT1 = "RT1"; RT0T1 = "RT0T1"; RC = "RC"; RCT0 = "RCT0"; RCT1 = "RCT1"; RCT0T1 = "RCT0T1"
    RS = "RS"; RST0 = "RST0"; RST1 = "RST1"; RST0T1 = "RST0T1"; RSC = "RSC"; RSCT0 = "RSCT0"; RSCT1 = "RSCT1"
    RSCT0T1 = "RSCT0T1"


def _desc(d):
    if d is None:
        return None
    return obj("GrB_DESC_" + d.value)


def init():
    """matrix.rs:116-185 (GxB_init NONBLOCKING + JIT control + LAGraph_Init)"""
    L = lib()
    check(L.GxB_init(0, None, None, None, None))
    check(L.GrB_Global_set_INT32(obj("GrB_GLOBAL"), 2, 7029))
    assert L.LAGraph_Init(None) == 0


def _u64arr(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _operands(ms, deltas):
    """(m, dp, dm, n): the handle arrays of operands `ms` and of their deltas, one (dp, dm) pair per operand (either may be None;
    `deltas` None: no pending writes).  Matrix objects or raw handles."""
    n = len(ms)
    deltas = [(None, None)] * n if deltas is None else list(deltas)
    assert len(deltas) == n, "one (dp, dm) pair per operand"
    arr = lambda xs: (C.c_void_p * max(1, n))(*[_handle(x) for x in xs])
    return arr(ms), arr([d[0] for d in deltas]), arr([d[1] for d in deltas]), n


class Matrix:
    """``Matrix<bool>`` (dtype=bool) or ``Matrix<u64>`` (dtype='u64')."""

    def __init__(self, nrows, ncols, dtype=bool, _handle=None):
        self.dtype = bool if dtype in (bool, "bool") else "u64"
        if _handle is not None:
            self.h = _handle
            return
        h = P()
        check(lib().GrB_Matrix_new(C.byref(h), obj("GrB_BOOL" if self.dtype is bool else "GrB_UINT64"), nrows, ncols))
        self.h = h
        # pin_sparse, matrix.rs:405-426
        check(lib().GrB_Matrix_set_INT32(self.h, GxB_SPARSE | GxB_HYPERSPARSE, GxB_SPARSITY_CONTROL))
        check(lib().GrB_Matrix_set_INT32(self.h, 0, GrB_STORAGE_ORIENTATION_HINT))

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and self.h.value:
                lib().GrB_Matrix_free(C.byref(self.h))
        except Exception:
            pass

    # ---- constructors -------------------------------------------------------------------------
    @staticmethod
    def import_csr(nrows, ncols, p, j, x=None, dtype=bool):
        p = np.ascontiguousarray(p, dtype=np.uint64)
        j = np.ascontiguousarray(j, dtype=np.uint32)
        xx = None if x is None else np.ascontiguousarray(x, dtype=np.uint64)
        h = P()
        dt = bool if dtype in (bool, "bool") else "u64"
        check(lib().B200_Matrix_import_CSR(C.byref(h), obj("GrB_BOOL" if dt is bool else "GrB_UINT64"), nrows, ncols,
                                           p.ctypes.data, j.ctypes.data if len(j) else None,
                                           None if xx is None else xx.ctypes.data, 0))
        return Matrix(nrows, ncols, dt, _handle=h)

    def export_csr(self):
        n, nnz = self.nrows(), self.nvals()
        p = np.empty(n + 1, np.uint64)
        j = np.empty(nnz, np.uint32)
        x = np.empty(nnz, np.uint64) if self.dtype != bool else None
        check(lib().B200_Matrix_export_CSR(self.h, p.ctypes.data, j.ctypes.data if nnz else None,
                                           None if x is None else x.ctypes.data, 0))
        return p.astype(np.int64), j, x

    def export_bitmap(self, out=None):
        """Row-major packed bitmap (B200_Matrix_export_bitmap): uint64[nrows, ceil(ncols/64)], bit (j & 63) of word j >> 6 of
        row i set iff (i, j) is an entry.  Returns (bitmap, nvals).  `out` may be a caller (pinned) buffer of that shape."""
        nr, nc = self.nrows(), self.ncols()
        wpr = (nc + 63) // 64
        if out is None:
            out = np.empty((nr, wpr), np.uint64)
        assert out.dtype == np.uint64 and out.size >= nr * wpr and out.flags.c_contiguous
        nv = U64()
        check(lib().B200_Matrix_export_bitmap(self.h, out.ctypes.data, wpr, C.byref(nv), 0))
        return out, nv.value

    def export_bitmap_async(self, out):
        """Non-blocking export_bitmap into `out` (pinned uint64[nrows, ceil(ncols/64)]): returns a ticket for `wait_ticket`;
        the copy runs on the library's second stream, so further mxm calls overlap it.  The matrix may be dropped at once."""
        nr, nc = self.nrows(), self.ncols()
        wpr = (nc + 63) // 64
        assert out.dtype == np.uint64 and out.size >= nr * wpr and out.flags.c_contiguous
        t = P()
        check(lib().B200_Matrix_export_bitmap_async(self.h, out.ctypes.data, wpr, C.byref(t)))
        return t

    def export_auto(self, out_bitmap=None):
        """The result hand-off a traversal operator makes: bitmap when the result is denser than one entry per 32 slots
        (1 bit per slot beats a 4-byte column index per entry), CSR otherwise -- the rule SuiteSparse applies when it
        switches a matrix to GxB_BITMAP.  Returns ("bitmap", bitmap, nvals) or ("csr", (p, j, x), nvals)."""
        nv = self.nvals()
        if nv * 32 > self.nrows() * self.ncols():
            bm, nv2 = self.export_bitmap(out_bitmap)
            return "bitmap", bm, nv2
        return "csr", self.export_csr(), nv

    def into_hyper(self):
        """matrix.rs:558-575"""
        check(lib().GrB_Matrix_set_INT32(self.h, GxB_HYPERSPARSE, GxB_SPARSITY_CONTROL))
        check(lib().GrB_Matrix_set_INT32(self.h, 0, GxB_HYPER_HASH))
        return self

    # ---- shape / status -----------------------------------------------------------------------
    def nrows(self):
        v = U64()
        check(lib().GrB_Matrix_nrows(C.byref(v), self.h))
        return v.value

    def ncols(self):
        v = U64()
        check(lib().GrB_Matrix_ncols(C.byref(v), self.h))
        return v.value

    def nvals(self):
        v = U64()
        check(lib().GrB_Matrix_nvals(C.byref(v), self.h))
        return v.value

    def pending(self):
        v = C.c_int32()
        check(lib().GrB_Matrix_get_INT32(self.h, C.byref(v), GxB_WILL_WAIT))
        return v.value == 1

    def sparsity_status(self):
        v = C.c_int32()
        check(lib().GrB_Matrix_get_INT32(self.h, C.byref(v), GxB_SPARSITY_STATUS))
        return {1: "hypersparse", 2: "sparse", 4: "bitmap", 8: "full"}.get(v.value, "unknown")

    def is_iso(self):
        v = C.c_bool()
        check(lib().GxB_Matrix_iso(C.byref(v), self.h))
        return v.value

    def memory_usage(self):
        v = C.c_size_t()
        check(lib().GxB_Matrix_memoryUsage(C.byref(v), self.h))
        return v.value

    def wait(self):
        check(lib().GrB_Matrix_wait(self.h, GrB_MATERIALIZE))

    def clear(self):
        check(lib().GrB_Matrix_clear(self.h))

    def resize(self, nrows, ncols):
        check(lib().GrB_Matrix_resize(self.h, nrows, ncols))

    def dup(self):
        h = P()
        check(lib().GrB_Matrix_dup(C.byref(h), self.h))
        return Matrix(0, 0, self.dtype, _handle=h)

    def grown(self, nrows, ncols):
        r0, c0 = self.nrows(), self.ncols()
        assert nrows >= r0 and ncols >= c0, f"grown must not shrink: {r0}x{c0} -> {nrows}x{ncols}"
        out = self.dup()
        if nrows != r0 or ncols != c0:
            out.resize(nrows, ncols)
        return out

    # ---- element access -----------------------------------------------------------------------
    def set(self, i, j, value=True):
        if self.dtype is bool:
            check(lib().GrB_Matrix_setElement_BOOL(self.h, bool(value), i, j))
        else:
            check(lib().GrB_Matrix_setElement_UINT64(self.h, int(value), i, j))

    def get(self, i, j):
        if self.dtype is bool:
            v = C.c_bool()
            info = lib().GrB_Matrix_extractElement_BOOL(C.byref(v), self.h, i, j)
        else:
            v = U64()
            info = lib().GrB_Matrix_extractElement_UINT64(C.byref(v), self.h, i, j)
        if info == 0:
            return v.value
        if info == 1:
            return None
        check(info)

    def contains(self, i, j):
        return lib().GxB_Matrix_isStoredElement(self.h, i, j) == 0

    def remove(self, i, j):
        check(lib().GrB_Matrix_removeElement(self.h, i, j))

    def build(self, rows, cols, vals=None):
        rows, cols = _u64arr(rows), _u64arr(cols)
        assert len(rows) == len(cols)
        if len(rows) == 0:
            return
        if self.dtype is bool:
            s = P()
            check(lib().GrB_Scalar_new(C.byref(s), obj("GrB_BOOL")))
            check(lib().GrB_Scalar_setElement_BOOL(s, True))
            try:
                check(lib().GxB_Matrix_build_Scalar(self.h, rows.ctypes.data, cols.ctypes.data, s, len(rows)))
            finally:
                lib().GrB_Scalar_free(C.byref(s))
        else:
            vals = _u64arr(vals)
            check(lib().GrB_Matrix_build_UINT64(self.h, rows.ctypes.data, cols.ctypes.data, vals.ctypes.data, len(rows),
                                                obj("GxB_ANY_UINT64")))

    # ---- bulk algebra -------------------------------------------------------------------------
    def lmxm(self, b):
        check(lib().GrB_mxm(self.h, None, None, obj("GxB_ANY_PAIR_BOOL"), self.h, b.h, None))

    def rmxm(self, b):
        check(lib().GrB_mxm(self.h, None, None, obj("GxB_ANY_PAIR_BOOL"), b.h, self.h, None))

    def mxm(self, a, b, mask=None, descriptor=None):
        check(lib().GrB_mxm(self.h, mask.h if mask is not None else None, None, obj("GxB_ANY_PAIR_BOOL"), a.h, b.h,
                            _desc(descriptor)))

    def delta_lmxm(self, m, dp, dm):
        """matrix.rs:1317-1402, statement for statement."""
        dp.wait()
        dm.wait()
        dp_nvals, dm_nvals = dp.nvals(), dm.nvals()
        if dp_nvals == 0 and dm_nvals == 0:
            self.lmxm(m)
            return
        nrows, ncols = self.nrows(), m.ncols()
        mask = None
        if dm_nvals > 0:
            mk = Matrix(nrows, ncols, bool)
            mk.mxm(self, dm)
            if mk.nvals() > 0:
                mask = mk
        accum = None
        if dp_nvals > 0:
            ac = Matrix(nrows, ncols, bool)
            ac.mxm(self, dp)
            if ac.nvals() > 0:
                accum = ac
        if mask is not None:
            self.mxm(self, m, mask, Descriptor.RSC)
        else:
            self.mxm(self, m)
        if accum is not None:
            self.element_wise_add(None, None, accum, None)

    def delta_lmxm_fused(self, m, dp, dm):
        """B200_Matrix_delta_lmxm: `delta_lmxm` as one call -- same result and flops; in device frontier form the dp / dm terms
        are applied to F*m in place, touching only the deltas' entries.  dp / dm may be None."""
        check(lib().B200_Matrix_delta_lmxm(self.h, m.h, None if dp is None else dp.h, None if dm is None else dm.h))

    def union_lmxm(self, ms, deltas=None):
        """B200_Matrix_union_lmxm: the union hop of `-[:R1|R2]->`, self <- self * U_t (ms[t] \\ dm_t) u dp_t, exact (no
        delta_lmxm over-masking, also for one operand).  `deltas`: one (dp, dm) pair per operand, either may be None."""
        check(lib().B200_Matrix_union_lmxm(self.h, *_operands(ms, deltas)))

    def element_wise_add(self, mask=None, a=None, b=None, descriptor=None):
        op = obj("GxB_ANY_BOOL") if self.dtype is bool else obj("GrB_SECOND_UINT64")
        check(lib().GrB_Matrix_eWiseAdd_BinaryOp(self.h, mask.h if mask is not None else None, None, op,
                                                 (a or self).h, (b or self).h, _desc(descriptor)))

    def element_wise_multiply(self, mask=None, a=None, b=None, descriptor=None):
        check(lib().GrB_Matrix_eWiseMult_Semiring(self.h, mask.h if mask is not None else None, None,
                                                  obj("GxB_ANY_PAIR_BOOL"), (a or self).h, (b or self).h, _desc(descriptor)))

    def intersection_nvals(self, b):
        t = Matrix(self.nrows(), self.ncols(), bool)
        check(lib().GrB_Matrix_eWiseMult_Semiring(t.h, None, None, obj("GxB_ANY_PAIR_BOOL"), self.h, b.h, None))
        return t.nvals()

    def set_pattern(self, mask, a, descriptor=None):
        check(lib().GrB_Matrix_apply(self.h, mask.h if mask is not None else None, obj("GxB_ANY_BOOL"), obj("GxB_ONE_BOOL"),
                                     a.h, _desc(descriptor)))

    def transpose(self):
        t = Matrix(self.ncols(), self.nrows(), self.dtype)
        check(lib().GrB_transpose(t.h, None, None, self.h, None))
        return t

    def remove_all(self, b):
        check(lib().GrB_transpose(self.h, b.h, None, self.h, obj("GrB_DESC_RCT0")))

    def select(self, mask, a):
        check(lib().GrB_transpose(self.h, mask.h, None, a.h, obj("GrB_DESC_RCT0")))

    # ---- iteration (matrix.rs:1471-1605: the reference's loop over the C iterator, verbatim) ----
    def iter(self, min_row=0, max_row=U64_MAX):
        L = lib()
        it = P()
        check(L.GxB_Iterator_new(C.byref(it)))
        try:
            check(L.GxB_rowIterator_attach(it, self.h, None))
            info = L.GxB_rowIterator_seekRow(it, min_row)
            while info == 1 and L.GxB_rowIterator_getRowIndex(it) < max_row:
                info = L.GxB_rowIterator_nextRow(it)
            depleted = info != 0 or L.GxB_rowIterator_getRowIndex(it) > max_row
            while not depleted:
                row, col = L.GxB_rowIterator_getRowIndex(it), L.GxB_rowIterator_getColIndex(it)
                item = (row, col) if self.dtype is bool else (row, col, L.GxB_Iterator_get_UINT64(it))
                if L.GxB_rowIterator_nextCol(it) != 0:
                    info = L.GxB_rowIterator_nextRow(it)
                    while info == 1 and L.GxB_rowIterator_getRowIndex(it) < max_row:
                        info = L.GxB_rowIterator_nextRow(it)
                    depleted = info != 0 or L.GxB_rowIterator_getRowIndex(it) > max_row
                yield item
        finally:
            L.GxB_Iterator_free(C.byref(it))

    def hyper_vector_count(self):
        if self.sparsity_status() != "hypersparse":
            return None
        L = lib()
        it = P()
        check(L.GxB_Iterator_new(C.byref(it)))
        check(L.GxB_rowIterator_attach(it, self.h, None))
        k = L.GxB_rowIterator_kount(it)
        L.GxB_Iterator_free(C.byref(it))
        return k

    def tuple_set(self):
        return set(self.iter())

    def extract_tuples(self):
        n = self.nvals()
        I, J = np.empty(n, np.uint64), np.empty(n, np.uint64)
        nv = U64(n)
        if self.dtype is bool:
            check(lib().GrB_Matrix_extractTuples_BOOL(I.ctypes.data, J.ctypes.data, None, C.byref(nv), self.h))
            return I, J, None
        X = np.empty(n, np.uint64)
        check(lib().GrB_Matrix_extractTuples_UINT64(I.ctypes.data, J.ctypes.data, X.ctypes.data, C.byref(nv), self.h))
        return I, J, X

    def extract_pairs(self, rows, cols):
        """Batched `get`: (found bool[n], values u64[n]) for the pairs (rows[t], cols[t]) -- ExpandInto's probe."""
        rows, cols = _u64arr(rows), _u64arr(cols)
        found = np.zeros(len(rows), np.uint8)
        vals = np.zeros(len(rows), np.uint64)
        check(lib().B200_Matrix_extract_pairs(self.h, rows.ctypes.data, cols.ctypes.data, len(rows), found.ctypes.data,
                                              vals.ctypes.data))
        return found.astype(bool), vals

    def digest(self):
        """(nvals, sum mix(key), sum mix(key + GOLD * position)) of the pattern in CSR order -- oracle.digest's twin."""
        d = np.zeros(3, np.uint64)
        check(lib().B200_Matrix_digest(self.h, d.ctypes.data))
        return d

    def prepare(self, want_transpose=True):
        check(lib().B200_Matrix_prepare(self.h, int(want_transpose)))
        return self

    def push_operand(self):
        """(ap, pperm, sorted) of a prepared square matrix: col_idx relabelled to hot-set positions (laid out by the rowptr), the
        vertex -> position table, and whether every row of ap is ascending -- B200_Matrix_push_operand."""
        ap = np.zeros(self.nvals(), np.uint32)
        pperm = np.zeros(self.ncols(), np.uint32)
        srt = C.c_int(0)
        check(lib().B200_Matrix_push_operand(self.h, ap.ctypes.data, pperm.ctypes.data, C.byref(srt)))
        return ap, pperm, bool(srt.value)


def rmat(scale, edge_factor=16, seed=1):
    h = P()
    check(lib().B200_Matrix_rmat(C.byref(h), scale, edge_factor, seed))
    return Matrix(0, 0, bool, _handle=h)


def bfs(A, src, max_level=-1, want_parent=True, deltas=None, dest=-1, info=None):
    """B200_bfs: (level, parent, edges traversed).  `A` may also be a list of operands (the relationship types algo.BFS names),
    and `deltas` one (dp, dm) pair per operand (either may be None): the BFS then walks the union of every (m \\ dm) u dp,
    exactly, through B200_bfs_delta, with the `dest` early exit and, given a B200_BfsInfo as `info`, what the run did."""
    if deltas is None and isinstance(A, Matrix) and dest < 0 and info is None:
        n = A.nrows()
        level = np.empty(n, np.int64)
        parent = np.empty(n, np.int64) if want_parent else None
        edges = U64()
        check(lib().B200_bfs(A.h, src, max_level, level.ctypes.data, None if parent is None else parent.ctypes.data, 0,
                             C.byref(edges)))
        return level, parent, edges.value
    ms = [A] if isinstance(A, Matrix) else list(A)
    ops = _operands(ms, deltas)
    n = ms[0].nrows()
    level = np.empty(n, np.int64)
    parent = np.empty(n, np.int64) if want_parent else None
    rec = BfsInfo() if info is None else info
    check(lib().B200_bfs_delta(*ops, src, max_level, dest, level.ctypes.data, None if parent is None else parent.ctypes.data, 0,
                               C.byref(rec)))
    return level, parent, rec.edges


def get_stat(name):
    return lib().B200_get_stat(name.encode())


def reset_stats():
    lib().B200_reset_stats()


def set_option(name, value):
    check(lib().B200_set_option(name.encode(), int(value)))


def sync():
    check(lib().B200_sync())


def wait_ticket(ticket):
    """B200_Ticket_wait: the buffer given to export_bitmap_async is complete when this returns."""
    check(lib().B200_Ticket_wait(C.byref(ticket)))


OUT_AUTO, OUT_BITMAP, OUT_CSR = 0, 1, 2


def traverse_batch(sources, hop_matrices, fmt=OUT_AUTO, out_bitmap=None, out_p=None, out_j=None, deltas=None):
    """B200_traverse_batch: the batched traversal an operator runs (cond_traverse.rs:600-608), host to host, as ONE C call.
    F(i, sources[i]) = 1, F <- F * hop_matrices[0] * ... ; the result lands in `out_bitmap` (uint64[nsrc, ceil(n/64)], pinned for
    overlapped copies) and / or (`out_p` uint64[nsrc+1], `out_j` uint32[capacity]).  Returns (flops, nvals or None, format).
    `deltas`: one (dp, dm) pair per hop (either may be None) -- hop h is then delta_lmxm by (hop_matrices[h], dp, dm), through
    B200_traverse_batch_delta.
    A hop given as a LIST of operands is a union hop (the types of `-[:R1|R2]->`, Matrix.union_lmxm), and its entry of `deltas`
    (if given) a list with one (dp, dm) pair per operand; any such hop sends the call through B200_traverse_batch_union."""
    sources = _u64arr(sources)
    nh = len(hop_matrices)
    nv, fl, chosen = U64(0), U64(0), C.c_int(0)
    wpr = out_bitmap.shape[1] if out_bitmap is not None else 0
    outs = (fmt, None if out_bitmap is None else out_bitmap.ctypes.data, wpr,
            None if out_p is None else out_p.ctypes.data, None if out_j is None else out_j.ctypes.data,
            0 if out_j is None else len(out_j), C.byref(nv), C.byref(fl), C.byref(chosen))
    if any(isinstance(h, (list, tuple)) for h in hop_matrices):
        assert deltas is None or len(deltas) == nh, "one deltas entry per hop"
        ms, pairs, nops, union = [], [], [], []
        for k, h in enumerate(hop_matrices):
            group = list(h) if isinstance(h, (list, tuple)) else [h]
            d = (None, None) if deltas is None else deltas[k]
            d = ([(None, None)] * len(group) if d is None else list(d)) if isinstance(h, (list, tuple)) else [d]
            assert len(d) == len(group), "one (dp, dm) pair per operand of a union hop"
            ms += group
            pairs += d
            nops.append(len(group))
            union.append(1 if isinstance(h, (list, tuple)) else 0)
        info = lib().B200_traverse_batch_union(sources.ctypes.data, len(sources), (C.c_int * nh)(*nops), (C.c_int * nh)(*union), nh,
                                               *_operands(ms, pairs)[:3], *outs)
    elif deltas is None:
        hs = (C.c_void_p * nh)(*[m.h for m in hop_matrices])
        info = lib().B200_traverse_batch(sources.ctypes.data, len(sources), hs, nh, *outs)
    else:
        assert len(deltas) == nh, "one (dp, dm) pair per hop"
        info = lib().B200_traverse_batch_delta(sources.ctypes.data, len(sources), *_operands(hop_matrices, deltas), *outs)
    if info == -103:                     # GrB_INSUFFICIENT_SPACE: nv holds the entries needed
        raise BufferError(f"out_j holds {0 if out_j is None else len(out_j)} entries, the result has {nv.value}")
    check(info)
    return fl.value, (None if nv.value == 2 ** 64 - 1 else nv.value), chosen.value


def traverse_to_host(sources, A, hops, out_bitmap, sub_batches=None):
    """Dense-result form of traverse_batch: `hops` times the same matrix, bitmap hand-off in 128-row slices whose device-to-host
    copies overlap the next slice's hops (the result transfer, not the GPU, bounds this call).  Returns the flops."""
    del sub_batches                      # the slicing lives in the library now
    return traverse_batch(sources, [A] * hops, OUT_BITMAP, out_bitmap=out_bitmap)[0]


def reach_batch(sources, A, max_hops=None, include_sources=False, deltas=None):
    """B200_reach_batch: `multi_source_reach` below as ONE C-ABI call (what a Rust operator would bind).  Returns (R, levels).
    `A` may also be a list of operands (the types of `-[:R1|R2*]->`), and `deltas` one (dp, dm) pair per operand (either may be
    None): the walked operand is then the union of every (m \\ dm) u dp, exactly, through B200_reach_batch_delta."""
    sources = _u64arr(sources)
    h, lv = P(), I64()
    hops = -1 if max_hops is None else int(max_hops)
    if deltas is None and isinstance(A, Matrix):
        check(lib().B200_reach_batch(C.byref(h), sources.ctypes.data, len(sources), A.h, hops, 1 if include_sources else 0,
                                     C.byref(lv)))
        return Matrix(0, 0, bool, _handle=h), lv.value
    ms = [A] if isinstance(A, Matrix) else list(A)
    check(lib().B200_reach_batch_delta(C.byref(h), sources.ctypes.data, len(sources), *_operands(ms, deltas), hops,
                                       1 if include_sources else 0, C.byref(lv)))
    return Matrix(0, 0, bool, _handle=h), lv.value


def adjacency(ms, deltas=None, n=None, keep=None, symmetric=False):
    """B200_adjacency_delta: the adjacency algo.pageRank / algo.WCC / algo.labelPropagation run on, as a new BOOL Matrix.  `ms`: one
    operand or a list, `deltas` one (dp, dm) pair per operand (either may be None); the result is the union of every (m \\ dm) u dp
    restricted to the vertices below `n` (default ncols) or, given `keep` (strictly ascending ids), to those, renumbered 0 ..
    len(keep) - 1.  `symmetric`: that union with its transpose."""
    ms = [ms] if isinstance(ms, Matrix) else list(ms)
    kp = None if keep is None else _u64arr(keep)
    h = P()
    check(lib().B200_adjacency_delta(C.byref(h), *_operands(ms, deltas), (ms[0].ncols() if ms else 0) if n is None else int(n),
                                     None if kp is None else kp.ctypes.data, 0 if kp is None else len(kp), 1 if symmetric else 0))
    return Matrix(0, 0, bool, _handle=h)


def multi_source_reach(sources, A, max_hops=None, include_sources=False):
    """Reachability from up to 1024 sources at once by level-synchronous mxm -- the multiplicity-insensitive core of a
    variable-length traversal `-[*1..k]->` with `emit_path = false` (cond_var_len_traverse.rs:196; SURVEY 8f-1) and of the
    BFS phase of allShortestPaths (all_shortest_paths.rs:7-25): row i of the result holds every vertex reachable from
    sources[i] by a walk of 1..max_hops edges (no bound: until no row finds a new vertex).
    Each level is C<!R, replace> = F*A (matrix.rs:1386: GrB_DESC_RSC, structural complement of the reached set) followed
    by R = R u F (matrix.rs:1398-1400) -- both stay in device frontier form.  Returns (R, levels run).
    With `include_sources` the zero-length walk (i, sources[i]) is part of R and never re-discovered."""
    sources = _u64arr(sources)
    nsrc, n = len(sources), A.ncols()
    rows = np.arange(nsrc, dtype=np.uint64)
    F = Matrix(nsrc, n, bool)
    F.build(rows, sources)
    R = Matrix(nsrc, n, bool)
    if include_sources:
        R.build(rows, sources)
    level = 0
    while max_hops is None or level < max_hops:
        if R.nvals():
            F.mxm(F, A, R, Descriptor.RSC)
        else:
            F.lmxm(A)
        if F.nvals() == 0:
            break
        R.element_wise_add(None, None, F, None)
        level += 1
    return R, level



DIR_OUT, DIR_IN, DIR_BOTH = 0, 1, 2
EDGES_ALL, EDGES_FIRST = 0, 1
TENSOR_LAYERS = ("m", "dp", "dm", "mt", "mt_dp", "mt_dm", "me", "me_dp", "me_dm")


class TensorLayers(C.Structure):
    """B200_TensorLayers (include/b200grb.h): one relationship type's nine layer handles"""
    _fields_ = [(k, P) for k in TENSOR_LAYERS]


def _handle(x):
    return None if x is None else (x.h if isinstance(x, Matrix) else x)


def _layers(types):
    """a B200_TensorLayers array, one entry per type: a sequence or dict of the nine layers in TENSOR_LAYERS order"""
    ls = (TensorLayers * max(1, len(types)))()
    for k, t in enumerate(types):
        vals = [t.get(name) for name in TENSOR_LAYERS] if isinstance(t, dict) else list(t) + [None] * (9 - len(t))
        for name, x in zip(TENSOR_LAYERS, vals):
            setattr(ls[k], name, _handle(x))
    return ls


def expand_edges(sources, types, dir=DIR_OUT, mode=EDGES_ALL, targets=None, capacity=None):
    """B200_expand_edges: the relationships of a batch of rows over relationship types, in one call.  `types`: one entry per type,
    a sequence or dict of the nine layers in TENSOR_LAYERS order (Matrix, raw handle or None; m required, mt for DIR_IN / DIR_BOTH).
    `targets` (same length as `sources`): row i covers only the neighbour targets[i] (ExpandInto).  Returns numpy arrays
    (p uint64[n+1], node uint32, edge uint64, type uint16, rev uint8); a result larger than `capacity` (default: a guess) is run
    once more into its size."""
    sources = _u64arr(sources)
    n = len(sources)
    if targets is not None:
        targets = _u64arr(targets)
        assert len(targets) == n, "one target per source"
    ls = _layers(types)
    cap = max(1024, 4 * n) if capacity is None else int(capacity)
    p, nv = np.zeros(n + 1, np.uint64), U64(0)
    for attempt in (0, 1):
        node, edge = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint64)
        typ, rev = np.zeros(max(cap, 1), np.uint16), np.zeros(max(cap, 1), np.uint8)
        info = lib().B200_expand_edges(sources.ctypes.data if n else None, None if targets is None else targets.ctypes.data, n, ls,
                                       len(types), dir, mode, p.ctypes.data, node.ctypes.data, edge.ctypes.data, typ.ctypes.data,
                                       rev.ctypes.data, cap, C.byref(nv))
        if info == -103 and attempt == 0:        # GrB_INSUFFICIENT_SPACE: nv holds the entries needed
            cap = nv.value
            continue
        check(info)
        break
    m = nv.value
    return p, node[:m], edge[:m], typ[:m], rev[:m]


PLAN_COMMITTED, PLAN_CANCEL, PLAN_MT_BASE, PLAN_EMPTIED, PLAN_DEMOTED, PLAN_M_HAS, PLAN_M_EQ = 1, 2, 4, 8, 16, 32, 64


def _plan(fn, t, a, b, c):
    a, b, c = _u64arr(a), _u64arr(b), _u64arr(c)
    n = len(a)
    assert len(b) == n and len(c) == n, "one entry per edge in each slice"
    rs, rd, rv, rf = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint8)
    mk, mi, mb = np.zeros(max(2 * n, 1), np.uint64), np.zeros(max(2 * n, 1), np.uint64), np.zeros(max(2 * n, 1), np.uint8)
    nr, nm = U64(0), U64(0)
    check(fn(_layers([t]), a.ctypes.data if n else None, b.ctypes.data if n else None, c.ctypes.data if n else None, n,
             rs.ctypes.data, rd.ctypes.data, rv.ctypes.data, rf.ctypes.data, C.byref(nr), mk.ctypes.data, mi.ctypes.data, mb.ctypes.data,
             C.byref(nm)))
    r, m = nr.value, nm.value
    return {"src": rs[:r], "dst": rd[:r], "val": rv[:r], "flags": rf[:r], "me_key": mk[:m], "me_id": mi[:m], "me_base": mb[:m].astype(bool)}


def insert_plan(t, srcs, dsts, ids):
    """B200_Tensor_insert_plan: the read phase of Tensor::set_all_from_slices over one type's layers `t` (a sequence or dict in
    TENSOR_LAYERS order, as expand_edges takes them).  Returns a dict of numpy arrays: the inline records (src, dst, val, flags) and
    the me entries (me_key, me_id, me_base)."""
    return _plan(lib().B200_Tensor_insert_plan, t, srcs, dsts, ids)


def remove_plan(t, ids, srcs, dsts):
    """B200_Tensor_remove_plan: the read phase of Tensor::remove_all's multi-edge path; the pair records (src, dst, val, flags) and
    the me entries, as insert_plan returns them."""
    return _plan(lib().B200_Tensor_remove_plan, t, ids, srcs, dsts)


def var_len_trails(starts, types, dir=DIR_OUT, min_hops=1, max_hops=None, dests=None, labels=(), mode="paths", tree_capacity=None,
                   capacity=None):
    """B200_var_len_trails: CondVarLenTraverse's trails from each start over relationship types (`types` as expand_edges takes
    them), in the reference's emission order.  max_hops None: unbounded.  dests: None or one int64 per start (< 0: none).  labels:
    destination labels, each a (m, dp, dm) triple of layers (Matrix, raw handle or None) or None for a label the graph lacks.
    mode "count": p only; "ends": p, end, hops; "paths": also the edges and nodes of every trail in walk order (trail k's edges are
    edges[E_k : E_k + hops[k]], E_k = sum(hops[:k]), its nodes nodes[E_k + k : E_k + k + hops[k] + 1]).  Returns a dict of numpy
    arrays.  Sized by a count call first unless `capacity` = (trails, path edges) is given."""
    starts = _u64arr(starts)
    n = len(starts)
    ds = None if dests is None else np.ascontiguousarray(dests, dtype=np.int64)
    assert ds is None or len(ds) == n, "one destination per start"
    ls = _layers(types)
    nl = len(labels)
    lm, ldp, ldm = (P * max(1, nl))(), (P * max(1, nl))(), (P * max(1, nl))()
    for k, lab in enumerate(labels):
        if lab is not None:
            lm[k], ldp[k], ldm[k] = (_handle(x) for x in (list(lab) + [None, None])[:3])
    mx = (1 << 64) - 1 if max_hops is None else int(max_hops)
    tc = (1 << 64) - 1 if tree_capacity is None else int(tree_capacity)
    p, nv, npth = np.zeros(n + 1, np.uint64), U64(0), U64(0)

    def call(end, hops, cap, pe, pn, pcap):
        return lib().B200_var_len_trails(starts.ctypes.data if n else None, None if ds is None else ds.ctypes.data, n, ls, len(types),
                                         dir, int(min_hops), mx, lm, ldp, ldm, nl, tc, p.ctypes.data, end, hops, cap, pe, pn, pcap,
                                         C.byref(nv), C.byref(npth))
    if mode == "count" or capacity is None:
        check(call(None, None, 0, None, None, 0))
        if mode == "count":
            return {"p": p, "nout": nv.value, "npath": npth.value}
        capacity = (nv.value, npth.value)
    cap, pcap = int(capacity[0]), int(capacity[1])
    end, hops = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint32)
    paths = mode == "paths"
    pe, pn = np.zeros(max(pcap, 1), np.uint64), np.zeros(max(pcap + cap, 1), np.uint32)
    check(call(end.ctypes.data, hops.ctypes.data, cap, pe.ctypes.data if paths else None, pn.ctypes.data if paths else None, pcap))
    m, q = nv.value, npth.value
    out = {"p": p, "end": end[:m], "hops": hops[:m], "nout": m, "npath": q}
    if paths:
        out["edges"], out["nodes"] = pe[:q], pn[:q + m]
    return out


def var_len_reach_both(starts, types, min_hops=1, max_hops=None):
    """B200_var_len_reach_both: the DISTINCT endpoints of the bidirectional pattern (a)-[*min_hops..max_hops]-(b), min_hops <= 1,
    from each start over relationship types (`types` as expand_edges takes them; mt required).  Row i of the returned BOOL Matrix
    (len(starts) x n) holds every b the trail DFS emits from starts[i]: each v != starts[i] within max_hops undirected edges, and
    starts[i] itself when min_hops == 0 or a cycle of at most max_hops relationships runs through it.  max_hops None: unbounded."""
    starts = _u64arr(starts)
    n = len(starts)
    h = P()
    check(lib().B200_var_len_reach_both(C.byref(h), starts.ctypes.data if n else None, n, _layers(types), len(types), int(min_hops),
                                        (1 << 64) - 1 if max_hops is None else int(max_hops)))
    return Matrix(0, 0, bool, _handle=h)


def shortest_path(src, dst, fwd, bwd, min_hops=1, max_hops=None, fwd_deltas=None, bwd_deltas=None):
    """B200_shortest_path: shortestPath((a)-[*min_hops..max_hops]->(b)) for the pairs (src[i], dst[i]).  `fwd` / `bwd`: the operands
    each side walks (a Matrix or a list), `fwd_deltas` / `bwd_deltas` one (dp, dm) pair per operand (either may be None).  Returns one
    entry per pair: the path's nodes from src to dst as a uint32 array, or None (Null).  max_hops None: unbounded."""
    src, dst = _u64arr(src), _u64arr(dst)
    assert len(src) == len(dst), "one dst per src"
    n = len(src)
    fwd = [fwd] if isinstance(fwd, Matrix) else list(fwd)
    bwd = [bwd] if isinstance(bwd, Matrix) else list(bwd)
    out_p = np.zeros(n + 1, np.uint64)
    cap = max(16, n * (min(31, (1 << 64) - 1 if max_hops is None else int(max_hops)) + 1))   # fits every path of up to 31 edges
    for _ in range(2):                               # a result larger than the first guess is rerun into its size
        nodes = np.zeros(cap, np.uint32)
        nn = U64(0)
        info = lib().B200_shortest_path(src.ctypes.data if n else None, dst.ctypes.data if n else None, n, *_operands(fwd, fwd_deltas),
                                        *_operands(bwd, bwd_deltas), int(min_hops), (1 << 64) - 1 if max_hops is None else int(max_hops),
                                        out_p.ctypes.data, nodes.ctypes.data, cap, C.byref(nn))
        if info != -103:
            break
        cap = nn.value
    check(info)
    return [nodes[out_p[i]:out_p[i + 1]].copy() if out_p[i + 1] > out_p[i] else None for i in range(n)]


def all_shortest_paths(src, dst, types, dir=DIR_OUT, max_hops=None, first=None, edge_capacity=None):
    """B200_all_shortest_paths: allShortestPaths((a)-[*..max_hops]->(b)) for the pairs (src[i], dst[i]) over relationship types
    (`types` as expand_edges takes them; mt required), dir DIR_OUT or DIR_BOTH; max_hops None: unbounded.  edge_capacity 0: count
    only; None: room for every path; else pairs fill from rank first[i] (None: 0) on until a path no longer fits.  Returns a dict
    of numpy arrays: count and len per pair, p (paths written, a prefix over pairs), edges and nodes (path k's edges are
    edges[E_k : E_k + len], E_k the edges of the paths before it; its nodes nodes[E_k + k : E_k + k + len + 1])."""
    src, dst = _u64arr(src), _u64arr(dst)
    assert len(src) == len(dst), "one dst per src"
    n = len(src)
    fs = None if first is None else _u64arr(first)
    ls = _layers(types)
    count, ln, p = np.zeros(max(1, n), np.uint64), np.zeros(max(1, n), np.uint32), np.zeros(n + 1, np.uint64)
    ne = U64(0)
    mh = (1 << 64) - 1 if max_hops is None else int(max_hops)

    def call(pe, pn, cap):
        check(lib().B200_all_shortest_paths(src.ctypes.data if n else None, dst.ctypes.data if n else None, n, ls, len(types), int(dir),
                                            mh, None if fs is None else fs.ctypes.data, count.ctypes.data, ln.ctypes.data, p.ctypes.data,
                                            None if pe is None else pe.ctypes.data, None if pn is None else pn.ctypes.data, cap,
                                            C.byref(ne)))
    if edge_capacity is None:
        call(None, None, 0)
        f = np.zeros(n, np.uint64) if fs is None else fs
        edge_capacity = int(sum(int(c - min(c, x)) * int(l) for c, x, l in zip(count[:n], f, ln[:n])))
    edges, nodes = np.zeros(max(1, edge_capacity), np.uint64), np.zeros(max(1, 2 * edge_capacity), np.uint32)
    if edge_capacity:
        call(edges, nodes, edge_capacity)
    else:
        call(None, None, 0)
    return {"count": count[:n].copy(), "len": ln[:n].copy(), "p": p, "edges": edges[:ne.value].copy(),
            "nodes": nodes[:ne.value + int(p[n])].copy()}
