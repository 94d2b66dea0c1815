"""ctypes binding of libb200grb.so -- the stub a reference maintainer would replace bindgen's
`extern "C"` block with (graph/src/graph/graphblas/mod.rs).  Fails loudly if the library is absent."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200GRB_LIB") or os.path.join(_HERE, "libb200grb.so")   # override: A/B builds of the same ABI

INFO = {0: "GrB_SUCCESS", 1: "GrB_NO_VALUE", 7089: "GxB_EXHAUSTED", -1: "GrB_UNINITIALIZED_OBJECT",
        -2: "GrB_NULL_POINTER", -3: "GrB_INVALID_VALUE", -4: "GrB_INVALID_INDEX", -5: "GrB_DOMAIN_MISMATCH",
        -6: "GrB_DIMENSION_MISMATCH", -7: "GrB_OUTPUT_NOT_EMPTY", -8: "GrB_NOT_IMPLEMENTED", -9: "GrB_ALREADY_SET",
        -101: "GrB_PANIC", -102: "GrB_OUT_OF_MEMORY", -103: "GrB_INSUFFICIENT_SPACE", -104: "GrB_INVALID_OBJECT",
        -105: "GrB_INDEX_OUT_OF_BOUNDS", -106: "GrB_EMPTY_OBJECT", -7001: "GxB_JIT_ERROR", -7002: "GxB_GPU_ERROR",
        -7003: "GxB_OUTPUT_IS_READONLY"}


class GrbError(RuntimeError):
    def __init__(self, info, msg=""):
        self.info = info
        super().__init__(f"{INFO.get(info, info)}: {msg}")


_lib = None
P = C.c_void_p
U64 = C.c_uint64
I64 = C.c_int64


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(this backend has no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    sig = {
        "GxB_init": [C.c_int, P, P, P, P], "GrB_init": [C.c_int], "GrB_finalize": [],
        "GrB_Global_set_INT32": [P, C.c_int32, C.c_int], "GxB_Global_Option_set_INT32": [C.c_int, C.c_int32],
        "GrB_Matrix_new": [C.POINTER(P), P, U64, U64], "GrB_Matrix_dup": [C.POINTER(P), P],
        "GrB_Matrix_free": [C.POINTER(P)], "GrB_Matrix_clear": [P], "GrB_Matrix_resize": [P, U64, U64],
        "GrB_Matrix_nrows": [C.POINTER(U64), P], "GrB_Matrix_ncols": [C.POINTER(U64), P],
        "GrB_Matrix_nvals": [C.POINTER(U64), P], "GrB_Matrix_set_INT32": [P, C.c_int32, C.c_int],
        "GrB_Matrix_get_INT32": [P, C.POINTER(C.c_int32), C.c_int], "GxB_Matrix_type": [C.POINTER(P), P],
        "GxB_Matrix_iso": [C.POINTER(C.c_bool), P], "GxB_Matrix_memoryUsage": [C.POINTER(C.c_size_t), P],
        "GxB_Matrix_fprint": [P, C.c_char_p, C.c_int, P], "GrB_Matrix_wait": [P, C.c_int],
        "GrB_Matrix_setElement_BOOL": [P, C.c_bool, U64, U64], "GrB_Matrix_setElement_UINT64": [P, U64, U64, U64],
        "GrB_Matrix_extractElement_BOOL": [C.POINTER(C.c_bool), P, U64, U64],
        "GrB_Matrix_extractElement_UINT64": [C.POINTER(U64), P, U64, U64],
        "GrB_Matrix_removeElement": [P, U64, U64], "GxB_Matrix_isStoredElement": [P, U64, U64],
        "GrB_Matrix_extractTuples_BOOL": [P, P, P, C.POINTER(U64), P],
        "GrB_Matrix_extractTuples_UINT64": [P, P, P, C.POINTER(U64), P],
        "GrB_Scalar_new": [C.POINTER(P), P], "GrB_Scalar_setElement_BOOL": [P, C.c_bool], "GrB_Scalar_free": [C.POINTER(P)],
        "GxB_Matrix_build_Scalar": [P, P, P, P, U64], "GrB_Matrix_build_UINT64": [P, P, P, P, U64, P],
        "GrB_Matrix_build_BOOL": [P, P, P, P, U64, P],
        "GrB_mxm": [P, P, P, P, P, P, P], "GrB_Matrix_eWiseAdd_BinaryOp": [P, P, P, P, P, P, P],
        "GrB_Matrix_eWiseMult_Semiring": [P, P, P, P, P, P, P], "GrB_transpose": [P, P, P, P, P],
        "GrB_Matrix_apply": [P, P, P, P, P, P],
        "GrB_Vector_new": [C.POINTER(P), P, U64], "GrB_Vector_free": [C.POINTER(P)], "GrB_Vector_size": [C.POINTER(U64), P],
        "GrB_Vector_nvals": [C.POINTER(U64), P], "GrB_Vector_setElement_BOOL": [P, C.c_bool, U64],
        "GrB_Vector_extractElement_INT64": [C.POINTER(I64), P, U64], "GrB_Vector_extractElement_BOOL": [C.POINTER(C.c_bool), P, U64],
        "GrB_Vector_extractTuples_INT64": [P, P, C.POINTER(U64), P], "GrB_Vector_extractTuples_BOOL": [P, P, C.POINTER(U64), P],
        "GrB_Vector_setElement_UINT64": [P, U64, U64], "GrB_Vector_removeElement": [P, U64], "GrB_Vector_clear": [P],
        "GrB_Vector_wait": [P, C.c_int], "GrB_Vector_resize": [P, U64],
        "GxB_Vector_Iterator_attach": [P, P, P], "GxB_Vector_Iterator_seek": [P, U64], "GxB_Vector_Iterator_next": [P],
        "GrB_Vector_setElement_FP64": [P, C.c_double, U64], "GrB_Vector_extractElement_FP64": [C.POINTER(C.c_double), P, U64],
        "GrB_Vector_extractTuples_FP64": [P, P, C.POINTER(U64), P],
        "GrB_Matrix_build_FP64": [P, P, P, P, U64, P], "GrB_Matrix_extractTuples_FP64": [P, P, P, C.POINTER(U64), P],
        "LAGraph_Cached_AT": [P, C.c_char_p], "LAGraph_Cached_OutDegree": [P, C.c_char_p],
        "LAGr_ConnectedComponents": [C.POINTER(P), P, C.c_char_p],
        "LAGraph_cdlp": [C.POINTER(P), P, C.c_int, C.c_char_p],
        "LAGr_PageRank": [C.POINTER(P), C.POINTER(C.c_int), P, C.c_float, C.c_float, C.c_int, C.c_char_p],
        "GrB_vxm": [P, P, P, P, P, P, P], "GrB_mxv": [P, P, P, P, P, P, P],
        "GxB_Iterator_new": [C.POINTER(P)], "GxB_Iterator_free": [C.POINTER(P)], "GxB_rowIterator_attach": [P, P, P],
        "GxB_rowIterator_seekRow": [P, U64], "GxB_rowIterator_nextRow": [P], "GxB_rowIterator_nextCol": [P],
        "LAGraph_Init": [C.c_char_p], "LAGraph_Finalize": [C.c_char_p], "LAGraph_New": [C.POINTER(P), C.POINTER(P), C.c_int, C.c_char_p],
        "LAGraph_Delete": [C.POINTER(P), C.c_char_p],
        "LAGr_BreadthFirstSearch_Extended": [C.POINTER(P), C.POINTER(P), P, U64, I64, I64, C.c_bool, C.c_char_p],
        "B200_Matrix_import_CSR": [C.POINTER(P), P, U64, U64, P, P, P, C.c_int],
        "B200_reach_batch": [C.POINTER(P), P, U64, P, I64, C.c_int, C.POINTER(I64)],
        "B200_reach_batch_delta": [C.POINTER(P), P, U64, P, P, P, C.c_int, I64, C.c_int, C.POINTER(I64)],
        "B200_Tensor_bulk_build": [C.POINTER(P), C.POINTER(C.POINTER(U64)), C.POINTER(C.POINTER(U64)), C.POINTER(U64), U64, U64, P, P, P, U64],
        "B200_Matrix_export_CSR": [P, P, P, P, C.c_int],
        "B200_Matrix_export_bitmap": [P, P, U64, C.POINTER(U64), C.c_int],
        "B200_Matrix_export_bitmap_async": [P, P, U64, C.POINTER(P)], "B200_Ticket_wait": [C.POINTER(P)],
        "B200_Matrix_device_view": [P, C.POINTER(P), C.POINTER(P), C.POINTER(P)],
        "B200_Matrix_digest": [P, P], "B200_Matrix_prepare": [P, C.c_int], "B200_Matrix_push_operand": [P, P, P, P], "B200_Matrix_rmat": [C.POINTER(P), C.c_int, U64, U64], "B200_sync": [], "B200_pool_trim": [],
        "B200_traverse_batch": [P, U64, P, C.c_int, C.c_int, P, U64, P, P, U64, C.POINTER(U64), C.POINTER(U64), C.POINTER(C.c_int)],
        "B200_traverse_batch_delta": [P, U64, P, P, P, C.c_int, C.c_int, P, U64, P, P, U64, C.POINTER(U64), C.POINTER(U64),
                                      C.POINTER(C.c_int)],
        "B200_Matrix_delta_lmxm": [P, P, P, P],
        "B200_Matrix_union_lmxm": [P, P, P, P, C.c_int],
        "B200_traverse_batch_union": [P, U64, P, P, C.c_int, P, P, P, C.c_int, P, U64, P, P, U64, C.POINTER(U64), C.POINTER(U64),
                                      C.POINTER(C.c_int)],
        "B200_expand_edges": [P, P, U64, P, C.c_int, C.c_int, C.c_int, P, P, P, P, P, U64, C.POINTER(U64)],
        "B200_set_option": [C.c_char_p, I64],
        "B200_Matrix_extract_pairs": [P, P, P, U64, P, P],
        "B200_Matrix_rmat_block": [C.POINTER(P), C.c_int, U64, U64, U64, U64, C.c_int],
        "B200_bfs": [P, U64, I64, P, P, C.c_int, C.POINTER(U64)],
        "B200_bfs_ex": [P, U64, I64, I64, P, P, C.c_int, P],
        "B200_bfs_delta": [P, P, P, C.c_int, U64, I64, I64, P, P, C.c_int, P],
        "B200_adjacency_delta": [C.POINTER(P), P, P, P, C.c_int, U64, P, U64, C.c_int],
        "B200_Tensor_insert_plan": [P, P, P, P, U64, P, P, P, P, C.POINTER(U64), P, P, P, C.POINTER(U64)],
        "B200_Tensor_remove_plan": [P, P, P, P, U64, P, P, P, P, C.POINTER(U64), P, P, P, C.POINTER(U64)],
        "B200_var_len_trails": [P, P, U64, P, C.c_int, C.c_int, U64, U64, P, P, P, C.c_int, U64, P, P, P, U64, P, P, U64,
                                C.POINTER(U64), C.POINTER(U64)],
        "B200_var_len_reach_both": [C.POINTER(P), P, U64, P, C.c_int, U64, U64],
        "B200_shortest_path": [P, P, U64, P, P, P, C.c_int, P, P, P, C.c_int, U64, U64, P, P, U64, C.POINTER(U64)],
        "B200_all_shortest_paths": [P, P, U64, P, C.c_int, C.c_int, U64, P, P, P, P, P, P, U64, C.POINTER(U64)],
        "B200_comm_unique_id": [P], "B200_comm_init": [C.POINTER(P), C.c_int, C.c_int, P], "B200_comm_free": [C.POINTER(P)],
        "B200_bfs_partitioned": [P, P, U64, U64, P, U64, I64, I64, P, P, C.c_int, P],
    }
    for name, args in sig.items():
        f = getattr(L, name)
        f.argtypes = args
        f.restype = C.c_int
    for name in ("GxB_rowIterator_kount", "GxB_rowIterator_getRowIndex", "GxB_rowIterator_getColIndex", "GxB_Iterator_get_UINT64",
                 "GxB_Vector_Iterator_getpmax", "GxB_Vector_Iterator_getp", "GxB_Vector_Iterator_getIndex"):
        f = getattr(L, name)
        f.argtypes = [P]
        f.restype = U64
    L.GxB_Iterator_get_BOOL.argtypes = [P]
    L.GxB_Iterator_get_BOOL.restype = C.c_bool
    L.B200_kernel_stats.argtypes = [C.c_char_p, C.POINTER(C.c_double), C.POINTER(U64), C.POINTER(U64)]
    L.B200_kernel_stats.restype = C.c_int
    L.B200_stream.restype = P
    L.B200_get_stat.argtypes = [C.c_char_p]
    L.B200_get_stat.restype = U64
    L.B200_reset_stats.restype = None
    L.B200_last_error.restype = C.c_char_p
    _lib = L
    return L


class BfsInfo(C.Structure):
    """B200_BfsInfo (include/b200grb.h)"""
    _fields_ = [("depth", U64), ("edges", U64), ("td_levels", U64), ("bu_levels", U64), ("sparse_levels", U64), ("exchanges", U64),
                ("exchanged_bytes", U64), ("device_ms", C.c_double), ("exchange_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def obj(name):
    """An exported data symbol holding an opaque handle (GrB_BOOL, GxB_ANY_PAIR_BOOL, GrB_DESC_RSC ...)."""
    return C.c_void_p.in_dll(lib(), name)


def check(info, ok=(0,)):
    if info not in ok:
        raise GrbError(info, (lib().B200_last_error() or b"").decode())
    return info
