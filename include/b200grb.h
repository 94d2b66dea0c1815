/*
 * b200grb.h -- C ABI of libb200grb.so, the H100-native (sm_90a) GraphBLAS traversal backend.
 *
 * Drop-in boundary (SURVEY.md 8b): FalkorDB links SuiteSparse:GraphBLAS through the bindgen
 * declarations in graph/src/graph/graphblas/mod.rs and the link line graph/build.rs:52-55.
 * Every declaration below mirrors the C signature mod.rs binds (file:line cited per entry), so
 * swapping `static=graphblas` for `dylib=b200grb` re-points the graph store's hot calls
 * (graph/src/graph/graphblas/matrix.rs) at this library.  All entry points return GrB_Info
 * (mod.rs:274-296); handles are opaque and owned by the library until *_free.
 *
 * Scope: the subset on the traversal path -- GrB_mxm over GxB_ANY_PAIR_BOOL with structural /
 * complemented / replace masks, eWiseAdd / eWiseMult / transpose (incl. the RCT0 masked copy) /
 * apply(ONE) for delta-matrix sync, build, element access, row iterators, wait, and the BFS entry
 * LAGr_BreadthFirstSearch_Extended.  Anything else returns GrB_NOT_IMPLEMENTED.  There is no CPU
 * fallback: bulk operations run on the GPU or fail with GxB_GPU_ERROR.
 *
 * B200_* entry points are extensions (zero-copy CSR hand-off, statistics, the synthetic RMAT input
 * generator) with no SuiteSparse counterpart; they play the role GxB_Container load/unload plays in
 * the reference (matrix.rs:428-546).
 */
#ifndef B200GRB_H
#define B200GRB_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef uint64_t GrB_Index; /* mod.rs:271 */

typedef enum { /* mod.rs:274-296 */
    GrB_SUCCESS = 0,
    GrB_NO_VALUE = 1,
    GxB_EXHAUSTED = 7089,
    GrB_UNINITIALIZED_OBJECT = -1,
    GrB_NULL_POINTER = -2,
    GrB_INVALID_VALUE = -3,
    GrB_INVALID_INDEX = -4,
    GrB_DOMAIN_MISMATCH = -5,
    GrB_DIMENSION_MISMATCH = -6,
    GrB_OUTPUT_NOT_EMPTY = -7,
    GrB_NOT_IMPLEMENTED = -8,
    GrB_ALREADY_SET = -9,
    GrB_PANIC = -101,
    GrB_OUT_OF_MEMORY = -102,
    GrB_INSUFFICIENT_SPACE = -103,
    GrB_INVALID_OBJECT = -104,
    GrB_INDEX_OUT_OF_BOUNDS = -105,
    GrB_EMPTY_OBJECT = -106,
    GxB_JIT_ERROR = -7001,
    GxB_GPU_ERROR = -7002,
    GxB_OUTPUT_IS_READONLY = -7003
} GrB_Info;

typedef enum { GrB_NONBLOCKING = 0, GrB_BLOCKING = 1 } GrB_Mode;
typedef enum { GrB_COMPLETE = 0, GrB_MATERIALIZE = 1 } GrB_WaitMode;   /* mod.rs:3032-3033 */
typedef enum { GrB_ROWMAJOR = 0, GrB_COLMAJOR = 1 } GrB_Orientation;   /* mod.rs:3006-3007 */

/* option fields used by the reference (mod.rs:2887-2963, 152) */
#define GrB_STORAGE_ORIENTATION_HINT 100
#define GxB_BURBLE 7019
#define GxB_JIT_C_CONTROL 7029
#define GxB_SPARSITY_STATUS 7034
#define GxB_SPARSITY_CONTROL 7036
#define GxB_HYPER_HASH 7048
#define GxB_WILL_WAIT 7076
#define GxB_NTHREADS 7086
/* sparsity bits (mod.rs:159-162) */
#define GxB_HYPERSPARSE 1
#define GxB_SPARSE 2
#define GxB_BITMAP 4
#define GxB_FULL 8

typedef struct GB_Type_opaque *GrB_Type;             /* mod.rs:316 */
typedef struct GB_UnaryOp_opaque *GrB_UnaryOp;       /* mod.rs:322 */
typedef struct GB_BinaryOp_opaque *GrB_BinaryOp;     /* mod.rs:328 */
typedef struct GB_Semiring_opaque *GrB_Semiring;     /* mod.rs:346 */
typedef struct GB_Descriptor_opaque *GrB_Descriptor; /* mod.rs:310 */
typedef struct GB_Scalar_opaque *GrB_Scalar;         /* mod.rs:352 */
typedef struct GB_Vector_opaque *GrB_Vector;         /* mod.rs:358 */
typedef struct GB_Matrix_opaque *GrB_Matrix;         /* mod.rs:364 */
typedef struct GB_Global_opaque *GrB_Global;         /* mod.rs:370 */
typedef struct GB_Iterator_opaque *GxB_Iterator;     /* mod.rs:383 */

/* exported data symbols (mod.rs:430-544, 721, 1301, 1547, 1643, 3001, 6852) */
extern GrB_Type GrB_BOOL, GrB_UINT64, GrB_INT64, GrB_FP64;
extern GrB_Semiring GxB_ANY_PAIR_BOOL;
/* the weighted / ranking corner of the path (north_star: "a stated fp tolerance for PLUS_TIMES weighted paths"): FP64 mxv / vxm */
extern GrB_Semiring GrB_PLUS_TIMES_SEMIRING_FP64, GxB_PLUS_SECOND_FP64;
extern GrB_BinaryOp GxB_ANY_BOOL, GrB_SECOND_UINT64, GxB_ANY_UINT64, GrB_PLUS_FP64;
extern GrB_UnaryOp GxB_ONE_BOOL;
extern const GrB_Global GrB_GLOBAL;
/* the 31 predefined descriptors: T0/T1 = transpose input 0/1, C = complement mask,
 * S = structural mask, R = replace output (matrix.rs:80-85, 313-351) */
extern GrB_Descriptor GrB_DESC_T1, GrB_DESC_T0, GrB_DESC_T0T1, GrB_DESC_C, GrB_DESC_CT1, GrB_DESC_CT0, GrB_DESC_CT0T1,
    GrB_DESC_S, GrB_DESC_ST1, GrB_DESC_ST0, GrB_DESC_ST0T1, GrB_DESC_SC, GrB_DESC_SCT1, GrB_DESC_SCT0, GrB_DESC_SCT0T1,
    GrB_DESC_R, GrB_DESC_RT1, GrB_DESC_RT0, GrB_DESC_RT0T1, GrB_DESC_RC, GrB_DESC_RCT1, GrB_DESC_RCT0, GrB_DESC_RCT0T1,
    GrB_DESC_RS, GrB_DESC_RST1, GrB_DESC_RST0, GrB_DESC_RST0T1, GrB_DESC_RSC, GrB_DESC_RSCT1, GrB_DESC_RSCT0,
    GrB_DESC_RSCT0T1;

/* ---- lifecycle (matrix.rs:116-221) ---- */
GrB_Info GxB_init(int mode, void *(*user_malloc)(size_t), void *(*user_calloc)(size_t, size_t),
                  void *(*user_realloc)(void *, size_t), void (*user_free)(void *)); /* mod.rs:7970 */
GrB_Info GrB_init(int mode);
GrB_Info GrB_finalize(void);                                                          /* mod.rs:7967 */
GrB_Info GrB_Global_set_INT32(GrB_Global g, int32_t value, int field);                /* mod.rs:10974 */
GrB_Info GxB_Global_Option_set_INT32(int field, int32_t value);                       /* mod.rs:15577 */

/* ---- matrix objects ---- */
GrB_Info GrB_Matrix_new(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols); /* mod.rs:9444 */
GrB_Info GrB_Matrix_dup(GrB_Matrix *C, GrB_Matrix A);                                    /* mod.rs:9452 */
GrB_Info GrB_Matrix_free(GrB_Matrix *A);                                                 /* mod.rs:15072 */
GrB_Info GrB_Matrix_clear(GrB_Matrix A);                                                 /* mod.rs:9476 */
GrB_Info GrB_Matrix_resize(GrB_Matrix C, GrB_Index nrows_new, GrB_Index ncols_new);      /* mod.rs:14055 */
GrB_Info GrB_Matrix_nrows(GrB_Index *nrows, GrB_Matrix A);                               /* mod.rs:9479 */
GrB_Info GrB_Matrix_ncols(GrB_Index *ncols, GrB_Matrix A);                               /* mod.rs:9485 */
GrB_Info GrB_Matrix_nvals(GrB_Index *nvals, GrB_Matrix A);                               /* mod.rs:9491 */
GrB_Info GrB_Matrix_set_INT32(GrB_Matrix A, int32_t value, int field);                   /* mod.rs:10713 */
GrB_Info GrB_Matrix_get_INT32(GrB_Matrix A, int32_t *value, int field);                  /* mod.rs:10230 */
GrB_Info GxB_Matrix_type(GrB_Type *type, GrB_Matrix A);                                  /* mod.rs:9503 */
GrB_Info GxB_Matrix_iso(bool *iso, GrB_Matrix A);                                        /* mod.rs:15103 */
GrB_Info GxB_Matrix_memoryUsage(size_t *size, GrB_Matrix A);                             /* mod.rs:9497 */
GrB_Info GxB_Matrix_fprint(GrB_Matrix A, const char *name, int pr, FILE *f);             /* mod.rs:14132 */
GrB_Info GrB_Matrix_wait(GrB_Matrix A, int waitmode);                                    /* mod.rs:11078 */

/* ---- element access (matrix.rs:1143-1172, 1248-1275, 731-737, 1035-1045) ---- */
GrB_Info GrB_Matrix_setElement_BOOL(GrB_Matrix C, bool x, GrB_Index i, GrB_Index j);       /* mod.rs:9685 */
GrB_Info GrB_Matrix_setElement_UINT64(GrB_Matrix C, uint64_t x, GrB_Index i, GrB_Index j); /* mod.rs:9749 */
GrB_Info GrB_Matrix_extractElement_BOOL(bool *x, GrB_Matrix A, GrB_Index i, GrB_Index j);  /* mod.rs:9797 */
GrB_Info GrB_Matrix_extractElement_UINT64(uint64_t *x, GrB_Matrix A, GrB_Index i, GrB_Index j); /* mod.rs:9861 */
GrB_Info GrB_Matrix_removeElement(GrB_Matrix C, GrB_Index i, GrB_Index j);                 /* mod.rs:9924 */
GrB_Info GxB_Matrix_isStoredElement(GrB_Matrix A, GrB_Index i, GrB_Index j);               /* mod.rs:9917 */
GrB_Info GrB_Matrix_extractTuples_BOOL(GrB_Index *I, GrB_Index *J, bool *X, GrB_Index *nvals, GrB_Matrix A);     /* mod.rs:9931 */
GrB_Info GrB_Matrix_extractTuples_UINT64(GrB_Index *I, GrB_Index *J, uint64_t *X, GrB_Index *nvals, GrB_Matrix A); /* mod.rs:10003 */

/* ---- build (matrix.rs:1186-1210, 1281-1303) ---- */
GrB_Info GrB_Scalar_new(GrB_Scalar *s, GrB_Type type);      /* mod.rs:8677 */
GrB_Info GrB_Scalar_setElement_BOOL(GrB_Scalar s, bool x);  /* mod.rs:8726 */
GrB_Info GrB_Scalar_free(GrB_Scalar *s);                    /* mod.rs:15066 */
GrB_Info GxB_Matrix_build_Scalar(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, GrB_Scalar scalar,
                                 GrB_Index nvals);          /* mod.rs:9659 */
GrB_Info GrB_Matrix_build_UINT64(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const uint64_t *X,
                                 GrB_Index nvals, GrB_BinaryOp dup); /* mod.rs:9589 */
GrB_Info GrB_Matrix_build_BOOL(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const bool *X, GrB_Index nvals,
                               GrB_BinaryOp dup);           /* mod.rs:9509 */

/* ---- bulk algebra: the hot calls ---- */
GrB_Info GrB_mxm(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Matrix A, GrB_Matrix B,
                 GrB_Descriptor desc);                      /* mod.rs:11162; matrix.rs:935,956,1346,1366,1386 */
GrB_Info GrB_Matrix_eWiseAdd_BinaryOp(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_BinaryOp add, GrB_Matrix A,
                                      GrB_Matrix B, GrB_Descriptor desc); /* mod.rs:11316; matrix.rs:862 */
GrB_Info GrB_Matrix_eWiseMult_Semiring(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_Semiring semiring,
                                       GrB_Matrix A, GrB_Matrix B, GrB_Descriptor desc); /* mod.rs:11228; matrix.rs:749,884 */
GrB_Info GrB_transpose(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_Matrix A,
                       GrB_Descriptor desc);                /* mod.rs:14013; matrix.rs:658,829,841 */
GrB_Info GrB_Matrix_apply(GrB_Matrix C, GrB_Matrix Mask, GrB_BinaryOp accum, GrB_UnaryOp op, GrB_Matrix A,
                          GrB_Descriptor desc);             /* mod.rs:12375; matrix.rs:913 */

/* ---- vectors (frontier / BFS outputs; graph/src/graph/graphblas/vector.rs:44-55) ---- */
GrB_Info GrB_Vector_new(GrB_Vector *v, GrB_Type type, GrB_Index n);
GrB_Info GrB_Vector_free(GrB_Vector *v);
GrB_Info GrB_Vector_size(GrB_Index *n, GrB_Vector v);
GrB_Info GrB_Vector_nvals(GrB_Index *nvals, GrB_Vector v);
GrB_Info GrB_Vector_setElement_BOOL(GrB_Vector v, bool x, GrB_Index i);     /* vector.rs:127, 507 */
GrB_Info GrB_Vector_setElement_UINT64(GrB_Vector w, uint64_t x, GrB_Index i); /* mod.rs:9158; vector.rs:442 */
GrB_Info GrB_Vector_removeElement(GrB_Vector v, GrB_Index i);                 /* mod.rs:9318; vector.rs:519 */
GrB_Info GrB_Vector_clear(GrB_Vector v);                                      /* mod.rs:8924; vector.rs:98 */
GrB_Info GrB_Vector_wait(GrB_Vector object, int waitmode);                    /* mod.rs:11072; vector.rs:134 */
GrB_Info GrB_Vector_resize(GrB_Vector w, GrB_Index nrows_new);                /* mod.rs:14062; vector.rs:494 */
/* vector iterator: positions 0 .. nvals-1 in ascending index order; seek / next return GxB_EXHAUSTED past the end
 * (mod.rs:14972-14997; vector.rs:553-594).  GxB_Iterator_get_UINT64 reads the current value. */
GrB_Info GxB_Vector_Iterator_attach(GxB_Iterator iterator, GrB_Vector v, GrB_Descriptor desc);
GrB_Index GxB_Vector_Iterator_getpmax(GxB_Iterator iterator);
GrB_Info GxB_Vector_Iterator_seek(GxB_Iterator iterator, GrB_Index p);
GrB_Info GxB_Vector_Iterator_next(GxB_Iterator iterator);
GrB_Index GxB_Vector_Iterator_getp(GxB_Iterator iterator);
GrB_Index GxB_Vector_Iterator_getIndex(GxB_Iterator iterator);
GrB_Info GrB_Vector_extractElement_INT64(int64_t *x, GrB_Vector v, GrB_Index i);
GrB_Info GrB_Vector_extractElement_BOOL(bool *x, GrB_Vector v, GrB_Index i);
GrB_Info GrB_Vector_extractTuples_INT64(GrB_Index *I, int64_t *X, GrB_Index *nvals, GrB_Vector v);
GrB_Info GrB_Vector_extractTuples_BOOL(GrB_Index *I, bool *X, GrB_Index *nvals, GrB_Vector v);
GrB_Info GrB_Vector_setElement_FP64(GrB_Vector w, double x, GrB_Index i);
GrB_Info GrB_Vector_extractElement_FP64(double *x, GrB_Vector v, GrB_Index i);
GrB_Info GrB_Vector_extractTuples_FP64(GrB_Index *I, double *X, GrB_Index *nvals, GrB_Vector v);  /* algo_procedures.rs: extract_vector_f64 */
GrB_Info GrB_Matrix_build_FP64(GrB_Matrix C, const GrB_Index *I, const GrB_Index *J, const double *X, GrB_Index nvals, GrB_BinaryOp dup);
GrB_Info GrB_Matrix_extractTuples_FP64(GrB_Index *I, GrB_Index *J, double *X, GrB_Index *nvals, GrB_Matrix A);
/* w<mask> = u*A / A*u: one frontier step over ANY_PAIR (mod.rs:11173, 11184); over GrB_PLUS_TIMES_SEMIRING_FP64 / GxB_PLUS_SECOND_FP64
 * the FP64 mxv (no mask; accum NULL or GrB_PLUS_FP64; fixed summation order, rel 1e-12 against the sequential oracle) */
GrB_Info GrB_vxm(GrB_Vector w, GrB_Vector mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Vector u, GrB_Matrix A,
                 GrB_Descriptor desc);
GrB_Info GrB_mxv(GrB_Vector w, GrB_Vector mask, GrB_BinaryOp accum, GrB_Semiring semiring, GrB_Matrix A, GrB_Vector u,
                 GrB_Descriptor desc);

/* ---- row iterator (matrix.rs:1471-1605) -- real symbols, as bindgen declares them ---- */
GrB_Info GxB_Iterator_new(GxB_Iterator *it);                                      /* mod.rs:14848 */
GrB_Info GxB_Iterator_free(GxB_Iterator *it);                                     /* mod.rs:15084 */
GrB_Info GxB_rowIterator_attach(GxB_Iterator it, GrB_Matrix A, GrB_Descriptor d); /* mod.rs:14875 */
GrB_Index GxB_rowIterator_kount(GxB_Iterator it);                                 /* mod.rs:14882 */
GrB_Info GxB_rowIterator_seekRow(GxB_Iterator it, GrB_Index row);                 /* mod.rs:14885 */
GrB_Info GxB_rowIterator_nextRow(GxB_Iterator it);                                /* mod.rs:14897 */
GrB_Info GxB_rowIterator_nextCol(GxB_Iterator it);                                /* mod.rs:14900 */
GrB_Index GxB_rowIterator_getRowIndex(GxB_Iterator it);                           /* mod.rs:14903 */
GrB_Index GxB_rowIterator_getColIndex(GxB_Iterator it);                           /* mod.rs:14906 */
uint64_t GxB_Iterator_get_UINT64(GxB_Iterator it);                                /* mod.rs:15024 */
bool GxB_Iterator_get_BOOL(GxB_Iterator it);

/* ---- serialization (matrix.rs:428-546 Encode/Decode via GxB_Container; vector.rs:150-420) ---- */
#define GrB_NAME 10                 /* mod.rs:2879 */
#define GxB_JIT_C_NAME 7041         /* mod.rs:2897 */
#define GxB_MAX_NAME_LEN 128        /* mod.rs:158 */
extern GrB_Type GrB_UINT32;         /* mod.rs:541 (type of the `i` payload vector when ncols <= 2^32) */
/* 608 bytes, field offsets as asserted in mod.rs:14165-14237; the reference copies the struct bytes into its RDB stream
 * (pointer fields are nulled and re-created on decode, matrix.rs:455-470). */
struct GxB_Container_struct {
    uint64_t nrows, ncols;
    int64_t nrows_nonempty, ncols_nonempty;
    uint64_t nvals;
    uint64_t u64_future[11];
    int32_t format, orientation, header_arena;
    uint32_t u32_future[13];
    GrB_Vector p, h, b, i, x;
    GrB_Vector vector_future[11];
    GrB_Matrix Y;
    GrB_Matrix matrix_future[15];
    bool iso, jumbled;
    bool bool_future[30];
    void *void_future[16];
};
typedef struct GxB_Container_struct *GxB_Container;                                            /* mod.rs:14238 */
GrB_Info GxB_Container_new(GxB_Container *Container);                                          /* mod.rs:14240 */
GrB_Info GxB_Container_free(GxB_Container *Container);                                         /* mod.rs:15081 */
/* A's content moves into the container's p/h/b/i/x vectors (row-major sparse or hypersparse, see grb_api.cu); A is left empty */
GrB_Info GxB_unload_Matrix_into_Container(GrB_Matrix A, GxB_Container Container, GrB_Descriptor desc);  /* mod.rs:14264 */
/* A takes type, dimensions and content from the container (validated: the payload may come from GRAPH.RESTORE) */
GrB_Info GxB_load_Matrix_from_Container(GrB_Matrix A, GxB_Container Container, GrB_Descriptor desc);    /* mod.rs:14250 */
/* full (dense) payload vectors <-> raw arrays; arrays handed out are allocated with GxB_init's malloc */
GrB_Info GxB_Vector_load(GrB_Vector V, void **X, GrB_Type type, uint64_t n, uint64_t X_memsize, int handling,
                         GrB_Descriptor desc);                                                  /* mod.rs:14278 */
GrB_Info GxB_Vector_unload(GrB_Vector V, void **X, GrB_Type *type, uint64_t *n, uint64_t *X_memsize, int *handling,
                           GrB_Descriptor desc);                                                /* mod.rs:14289 */
/* opaque blob of a (sparse) vector: Tensor's multi-edge id lists (vector.rs:150-195); round-trips through this library only */
GrB_Info GxB_Vector_serialize(void **blob_handle, GrB_Index *blob_size, GrB_Vector u, GrB_Descriptor desc);   /* mod.rs:14717 */
GrB_Info GxB_Vector_deserialize(GrB_Vector *w, GrB_Type type, const void *blob, GrB_Index blob_size,
                                GrB_Descriptor desc);                                           /* mod.rs:14768 */
GrB_Info GrB_Type_get_String(GrB_Type type, char *value, int field);                            /* mod.rs:10503 */
GrB_Info GxB_Type_from_name(GrB_Type *type, const char *type_name);                             /* mod.rs:8075 */

/* ---- LAGraph subset (lagraph_bindings.rs:160-188, lagraphx_bindings.rs:585-594) ---- */
typedef enum { LAGraph_ADJACENCY_UNDIRECTED = 0, LAGraph_ADJACENCY_DIRECTED = 1, LAGraph_KIND_UNKNOWN = -1 } LAGraph_Kind;
typedef struct LAGraph_Graph_struct {
    GrB_Matrix A;
    LAGraph_Kind kind;
    GrB_Matrix AT;
    GrB_Vector out_degree, in_degree;
    int is_symmetric_structure;
    int64_t nself_edges;
    GrB_Scalar emin;
    int emin_state;
    GrB_Scalar emax;
    int emax_state;
} *LAGraph_Graph;
int LAGraph_Init(char *msg);
int LAGraph_Finalize(char *msg);
int LAGraph_New(LAGraph_Graph *G, GrB_Matrix *A, LAGraph_Kind kind, char *msg);
int LAGraph_Delete(LAGraph_Graph *G, char *msg);
int LAGr_BreadthFirstSearch_Extended(GrB_Vector *level, GrB_Vector *parent, LAGraph_Graph G, GrB_Index src,
                                     int64_t max_level, int64_t dest, bool many_expected, char *msg);
/* algo.pageRank (algo_procedures.rs:744-752; lagraph_bindings.rs:549-558): FP64 on the device, centrality = full GrB_FP64 vector */
int LAGraph_Cached_AT(LAGraph_Graph G, char *msg);
int LAGraph_Cached_OutDegree(LAGraph_Graph G, char *msg);
int LAGr_PageRank(GrB_Vector *centrality, int *iters, LAGraph_Graph G, float damping, float tol, int itermax, char *msg);
/* algo.WCC (algo_procedures.rs:838-846; lagraph_bindings.rs:521-526): component(i) = smallest vertex id of i's component (dense) */
int LAGr_ConnectedComponents(GrB_Vector *component, LAGraph_Graph G, char *msg);
/* algo.labelPropagation (algo_procedures.rs:1232-1237; lagraphx_bindings.rs:218-223): label(i) after <= itermax synchronous rounds
   of "most frequent neighbour label, smallest on ties" from label(i) = i (LDBC Graphalytics CDLP); full GrB_UINT64 vector */
int LAGraph_cdlp(GrB_Vector *CDLP_handle, LAGraph_Graph G, int itermax, char *msg);

/* ---- B200 extensions ---- */
#define B200_LOC_HOST 0
#define B200_LOC_DEVICE 1
/* Import a CSR (rowptr u64[nrows+1], col u32[nnz] ascending per row, val u64[nnz] or NULL) from host
 * or device memory; arrays are copied.  Plays the role of GxB_load_Matrix_from_Container. */
GrB_Info B200_Matrix_import_CSR(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols, const uint64_t *Ap,
                                const uint32_t *Aj, const uint64_t *Ax, int location);
/* Export into caller buffers sized by GrB_Matrix_nrows / nvals (Ax may be NULL). */
GrB_Info B200_Matrix_export_CSR(GrB_Matrix A, uint64_t *Ap, uint32_t *Aj, uint64_t *Ax, int location);
/* Export as a row-major packed bitmap: word `bits_out[i * words_per_row + (j >> 6)]` has bit (j & 63) set iff A(i,j) is an
 * entry; words_per_row must be ceil(ncols / 64) and every word of the nrows x words_per_row array is written.  The
 * interchange format for dense results (SuiteSparse keeps such matrices in GxB_BITMAP form and exports them with
 * GxB_Matrix_export_BitmapR; this is the 1-bit-per-slot equivalent): a frontier chain result that is still in device
 * bit-matrix form is exported without ever building its CSR.  Cheaper than CSR when nvals * 32 > nrows * ncols. */
GrB_Info B200_Matrix_export_bitmap(GrB_Matrix A, uint64_t *bits_out, uint64_t words_per_row, uint64_t *nvals_out, int location);
/* Same hand-off without blocking: the device-to-host copy runs on a second stream, so the caller can submit the next
 * batch's GrB_mxm calls while it is in flight (bits_out should be pinned).  A may be modified or freed right away; bits_out
 * is complete once B200_Ticket_wait returns.  Every ticket must be waited on exactly once. */
typedef struct B200_Ticket_opaque *B200_Ticket;
GrB_Info B200_Matrix_export_bitmap_async(GrB_Matrix A, uint64_t *bits_out, uint64_t words_per_row, B200_Ticket *ticket);
GrB_Info B200_Ticket_wait(B200_Ticket *ticket);
/* Borrow the device-resident CSR (valid until A is next modified or freed). */
/* digest3 = { nvals, sum mix(row << 32 | col), sum mix(key + GOLD * (CSR position + 1)) }: a multi-GB result is compared with the
 * oracle's through three numbers; sensitive to any changed entry and to the order inside a row */
GrB_Info B200_Matrix_digest(GrB_Matrix A, uint64_t *digest3);
GrB_Info B200_Matrix_device_view(GrB_Matrix A, const uint64_t **Ap, const uint32_t **Aj, const uint64_t **Ax);
/* Pre-build the cached transpose mirror used by the pull direction (done lazily otherwise). */
GrB_Info B200_Matrix_prepare(GrB_Matrix A, int want_transpose);
/* The CSR push's operand of a prepared square matrix, for inspection: ap_out[nvals] = col_idx relabelled to hot-set positions,
 * laid out by A's rowptr; pperm_out[ncols] = vertex -> position; *sorted = every row of ap ascending (the sliced push's
 * condition).  Either array may be NULL.  GrB_INVALID_VALUE when the matrix has no such table. */
GrB_Info B200_Matrix_push_operand(GrB_Matrix A, uint32_t *ap_out, uint32_t *pperm_out, int *sorted);
/* Synthetic Graph500-style RMAT adjacency (a,b,c,d=.57,.19,.19,.05), dedupe + no self loops, built on
 * the device.  Benchmark / test input only. */
GrB_Info B200_Matrix_rmat(GrB_Matrix *A, int scale, uint64_t edge_factor, uint64_t seed);
/* Row block [lo,hi) of B200_Matrix_rmat's matrix ((hi-lo) x 2^scale, rows local-indexed); by_col == 1 gives the same
 * block of the TRANSPOSE, by_col == 2 of the symmetrised strictly-lower-triangular matrix L = tril(A u A') (config 4).  Every rank regenerates the counter-based edge stream and keeps what it owns. */
GrB_Info B200_Matrix_rmat_block(GrB_Matrix *A, int scale, uint64_t edge_factor, uint64_t seed, uint64_t lo, uint64_t hi,
                                int by_col);

/* GRAPH.BULK's edge load into an EMPTY relationship tensor (src/commands/bulk_insert.rs:497 -> graph.rs:2062 ->
 * Tensor::set_all_from_slices, tensor.rs:333-447) as one device-side build: *fwd = the forward UINT64 matrix (value = the pair's
 * edge id, or UINT64_MAX = tensor.rs:206's MULTI_EDGE when the pair has several edges); *multi_keys / *multi_ids = (src << 32 | dst,
 * edge id) for every edge of every multi-edge pair, sorted by (key, id) -- the entries of `me`.  The two arrays come from GxB_init's
 * malloc (NULL when *nmulti == 0) and are the caller's to free. */
GrB_Info B200_Tensor_bulk_build(GrB_Matrix *fwd, GrB_Index **multi_keys, GrB_Index **multi_ids, GrB_Index *nmulti, GrB_Index nrows,
                                GrB_Index ncols, const GrB_Index *srcs, const GrB_Index *dsts, const GrB_Index *ids, GrB_Index n);
/* Batched point lookup: found[t] = 1 (and values[t] = A(I[t],J[t]) when `values` is non-NULL) iff the entry is stored.
 * ExpandInto's per-row Tensor::get (graph/src/runtime/ops/expand_into.rs:195-249 -> GrB_Matrix_extractElement_UINT64)
 * for a whole 1024-row batch in one device call; host arrays in, host arrays out. */
GrB_Info B200_Matrix_extract_pairs(GrB_Matrix A, const GrB_Index *I, const GrB_Index *J, GrB_Index n, uint8_t *found,
                                   uint64_t *values);
/* The coalesced traversal of CondTraverseOp::expand_batch as one call (cond_traverse.rs:600-608, 1264-1285): F(i, sources[i]) = 1,
 * F <- F * hops[0] * ... * hops[nhops-1] over GxB_ANY_PAIR_BOOL (square, equally sized operands), result rows to host memory as a
 * packed row-major bitmap (128-row slices, copies overlapped with the next slice's hops), as CSR, or whichever moves fewer bytes. */
#define B200_OUT_AUTO 0
#define B200_OUT_BITMAP 1
#define B200_OUT_CSR 2
GrB_Info B200_traverse_batch(const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *hops, int nhops, int format,
                             uint64_t *out_bits, uint64_t words_per_row, uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity,
                             uint64_t *nvals_out, uint64_t *flops_out, int *format_out);
/* delta_lmxm (matrix.rs:1317-1402) as one call, for an operand with pending writes held as base m plus deltas dp (added) and dm
 * (deleted): F <- (F*m AND NOT F*dm) OR F*dp over GxB_ANY_PAIR_BOOL, the reference's three-mxm-plus-eWiseAdd composition with its
 * over-masking ((i,j) is dropped whenever a deleted edge reaches j from row i).  Holds for arbitrary deltas; dp / dm may be NULL or
 * empty; values are ignored (m and dp may be UINT64); pending tuples of dp / dm are finished first.  In device frontier form the
 * delta terms touch only the deltas' entries; otherwise the composition runs.  last_flops = flops(F*m) + flops(F*dp) + flops(F*dm). */
GrB_Info B200_Matrix_delta_lmxm(GrB_Matrix F, GrB_Matrix m, GrB_Matrix dp, GrB_Matrix dm);
/* B200_traverse_batch over operands with pending writes: hop h is B200_Matrix_delta_lmxm(F, m[h], dp[h], dm[h]).  dp / dm may be
 * NULL arrays or hold NULL entries (clean hops); outputs and formats as B200_traverse_batch. */
GrB_Info B200_traverse_batch_delta(const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *m, const GrB_Matrix *dp,
                                   const GrB_Matrix *dm, int nhops, int format, uint64_t *out_bits, uint64_t words_per_row,
                                   uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity, uint64_t *nvals_out, uint64_t *flops_out,
                                   int *format_out);
/* The union hop of a fixed-length hop over several relationship types (MATCH (a)-[:R1|R2]->(b); CondTraverseOp's
 * build_relationship_matrix_unrestricted, graph.rs:2520-2550): F <- F * U_t (m[t] \ dm[t]) u dp[t] over GxB_ANY_PAIR_BOOL, exact
 * (no delta_lmxm over-masking), also for nops == 1.  Pattern only (m / dp may be UINT64, dm BOOL; within a type dp wins over dm; an
 * entry one type contributes survives another type's dm).  dp / dm may be NULL arrays or hold NULL entries.  Every operand and delta
 * is square of one size n = ncols(F) (else GrB_DIMENSION_MISMATCH); nops < 1 is GrB_INVALID_VALUE; host-resident operands are
 * GrB_NOT_IMPLEMENTED; with no device GxB_GPU_ERROR comes back before any host work.
 * last_flops = sum_t flops(F*m[t]) + flops(F*dp[t]). */
GrB_Info B200_Matrix_union_lmxm(GrB_Matrix F, const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops);
/* B200_traverse_batch over hop groups.  Operands are hop-major: hop h owns hop_nops[h] consecutive entries of m / dp / dm.
 * hop_union[h] == 0: a delta hop (hop_nops[h] must be 1), B200_Matrix_delta_lmxm; else a union hop, B200_Matrix_union_lmxm over
 * its operands.  Outputs, formats, GrB_INSUFFICIENT_SPACE and flops as B200_traverse_batch; operand errors as
 * B200_Matrix_union_lmxm.  hop_nops == 1 and hop_union == 0 everywhere is B200_traverse_batch_delta. */
GrB_Info B200_traverse_batch_union(const GrB_Index *sources, GrB_Index nsrc, const int *hop_nops, const int *hop_union, int nhops,
                                   const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int format, uint64_t *out_bits,
                                   uint64_t words_per_row, uint64_t *out_p, uint32_t *out_j, uint64_t out_j_capacity,
                                   uint64_t *nvals_out, uint64_t *flops_out, int *format_out);
/* Multi-source reachability in one call (SURVEY 8f-1: CondVarLenTraverse with emit_path = false, cond_var_len_traverse.rs:196;
 * AllShortestPaths' BFS phase, all_shortest_paths.rs:7-25): row i of *reached (new nsrc x n BOOL matrix) = the vertices reachable
 * from sources[i] by 1..max_hops edges of the square matrix A (max_hops < 0: to the fixed point); include_sources adds the
 * zero-length walk.  Levels are F<!R,replace,struct> = F*A then R = R u F, in device frontier form; *levels_out = levels run. */
GrB_Info B200_reach_batch(GrB_Matrix *reached, const GrB_Index *sources, GrB_Index nsrc, GrB_Matrix A, int64_t max_hops,
                          int include_sources, int64_t *levels_out);
/* B200_reach_batch over relationship tensors with pending writes: the walked operand is A = U_t (m[t] \ dm[t]) u dp[t], pattern
 * only (m / dp may be UINT64, dm BOOL; where dp and dm hold the same entry dp wins; dm entries outside m have no effect).  Exact:
 * a vertex stays reachable while any remaining edge reaches it (no delta_lmxm over-masking).  dp / dm may be NULL arrays or hold
 * NULL entries.  Every operand and delta is square of one size n (else GrB_DIMENSION_MISMATCH); nops < 1 is GrB_INVALID_VALUE;
 * host-resident operands are GrB_NOT_IMPLEMENTED.  One operand without deltas runs exactly B200_reach_batch. */
GrB_Info B200_reach_batch_delta(GrB_Matrix *reached, const GrB_Index *sources, GrB_Index nsrc, const GrB_Matrix *m,
                                const GrB_Matrix *dp, const GrB_Matrix *dm, int nops, int64_t max_hops, int include_sources,
                                int64_t *levels_out);
/* The layers of one relationship type's Tensor (tensor.rs:184-259), as B200_expand_edges reads them.  m / dp: forward UINT64 layers
 * (value = the pair's edge id, or UINT64_MAX = MULTI_EDGE), dm BOOL; mt / mt_dp / mt_dm: the maintained transpose, BOOL; me / me_dp
 * / me_dm: the multi-edge store (2^60 x 2^60 BOOL, row = src << 32 | dst, column = edge id).  Every layer but m may be NULL. */
typedef struct {
    GrB_Matrix m, dp, dm;
    GrB_Matrix mt, mt_dp, mt_dm;
    GrB_Matrix me, me_dp, me_dm;
} B200_TensorLayers;
#define B200_DIR_OUT 0
#define B200_DIR_IN 1
#define B200_DIR_BOTH 2
#define B200_EDGES_ALL 0   /* one entry per relationship (emit_relationship) */
#define B200_EDGES_FIRST 1 /* one entry per (row, direction, neighbour): the first id (bind_edge) */
/* The relationships of a batch of rows over ntypes relationship types, in one call (CondTraverse's expand_row / bind_edge,
 * ExpandInto's Tensor::get probes).  The value of a pair in one type is Tensor::eff_get's: dp if present, else none if dm holds
 * it, else m; a MULTI_EDGE value stands for the key's ids in (me \ me_dm) u me_dp, ascending.
 * Row i covers out_p[i] .. out_p[i+1] of out_node (the neighbour), out_edge (the id), out_type (index into types) and out_rev:
 *  - B200_DIR_OUT: the effective out-neighbours d of sources[i] over the types;
 *  - B200_DIR_IN: the in-neighbours k from each type's effective transpose row, ids looked up at forward (k, sources[i]);
 *  - B200_DIR_BOTH: the forward block, then the reverse block without k == sources[i] (out_rev = 1 marks reverse entries);
 *  - inside a block: neighbour ascending, then type index, then id.
 * targets non-NULL: row i covers only the neighbour targets[i] (ExpandInto).  B200_EDGES_FIRST keeps, per (row, block,
 * neighbour), the first entry of that order.  out_type / out_rev may be NULL.  out_p (n + 1 entries) is written in every case;
 * the entries only when they fit out_capacity, else GrB_INSUFFICIENT_SPACE with *nout = the entries needed.
 * Errors: ntypes outside 1 .. 65536, dir or mode out of range GrB_INVALID_VALUE; m not UINT64 (or dp not UINT64) GrB_DOMAIN_MISMATCH; forward and
 * transpose layers not square of one size n GrB_DIMENSION_MISMATCH; an id >= n GrB_INVALID_INDEX; mt NULL under DIR_IN / DIR_BOTH
 * GrB_NULL_POINTER; host-resident forward or transpose layers GrB_NOT_IMPLEMENTED (the me layers are host-resident: their stores
 * are uploaded once and cached with the handle until it changes); with no device GxB_GPU_ERROR before any host work. */
GrB_Info B200_expand_edges(const GrB_Index *sources, const GrB_Index *targets, GrB_Index n, const B200_TensorLayers *types,
                           int ntypes, int dir, int mode, uint64_t *out_p, uint32_t *out_node, uint64_t *out_edge,
                           uint16_t *out_type, uint8_t *out_rev, uint64_t out_capacity, uint64_t *nout);
/* CondVarLenTraverse's trails (cond_var_len_traverse.rs:152-386) from each starts[i], over ntypes tensors' live layers: every
 * relationship-unique path of min_hops .. max_hops edges, in the reference's emission order.  Adjacency per node is
 * Graph::get_node_relationships_by_type's (graph.rs:1797-1835): types in order; per type the outgoing half (neighbour ascending,
 * ids ascending), then the incoming half (source ascending); under Both a self-loop once, in the outgoing half.  Per start: the
 * 0-hop emission (min_hops == 0), then per frame its emitting edges in adjacency order, then the frames of its continuing edges in
 * reverse adjacency order (a DFS stack).  Starts come out in input order.
 * dir: B200_DIR_OUT (forward), B200_DIR_IN (reversed), B200_DIR_BOTH (bidirectional; the reference never combines it with
 * reversed, :534).  max_hops = UINT64_MAX: unbounded.  dests NULL or dests[i] < 0: no fixed destination.  Destination labels:
 * nlabels triples (lab_m, lab_dp, lab_dm), the label's diagonal being (m \ dm) u dp; a NULL lab_m is a label the graph lacks:
 * nothing emits.  lab_dp / lab_dm may be NULL arrays or hold NULL entries.
 * out_p[nstarts + 1] is always written (but see tree_capacity): trails of start i are out_p[i] .. out_p[i+1], in the reference's
 * emission order.  out_end (the node the walk ends at) and out_hops; out_end NULL: count only.  With path_edge / path_node the
 * trail itself in walk order from the start: trail k's edges are path_edge[E_k .. E_k + h_k), E_k = sum_{j<k} h_j, and its nodes
 * are path_node[E_k + k .. E_k + k + h_k] (path_node holds *npath + *nout entries).
 * Entries are written only when they fit: out_capacity trails and path_capacity edges.  Otherwise GrB_INSUFFICIENT_SPACE, with
 * *nout / *npath = what is needed.
 * If the stored trail tree (every trail shorter than max_hops) would exceed tree_capacity entries: GrB_INSUFFICIENT_SPACE with
 * *nout = *npath = UINT64_MAX, nothing written.
 * Errors follow B200_expand_edges (types' layers, ntypes, dir); nlabels < 0 GrB_INVALID_VALUE; a start or destination >= n
 * GrB_INVALID_INDEX; label layers not n x n GrB_DIMENSION_MISMATCH, host-resident GrB_NOT_IMPLEMENTED; out_end without out_hops, or
 * path_edge without path_node, GrB_NULL_POINTER.  nstarts == 0 or min_hops > max_hops: success with no device work.  No layer
 * changes, apart from finishing pending tuples; no base is downloaded. */
GrB_Info B200_var_len_trails(const GrB_Index *starts, const int64_t *dests, GrB_Index nstarts, const B200_TensorLayers *types,
                             int ntypes, int dir, uint64_t min_hops, uint64_t max_hops, const GrB_Matrix *lab_m,
                             const GrB_Matrix *lab_dp, const GrB_Matrix *lab_dm, int nlabels, uint64_t tree_capacity,
                             uint64_t *out_p, uint32_t *out_end, uint32_t *out_hops, uint64_t out_capacity,
                             uint64_t *path_edge, uint32_t *path_node, uint64_t path_capacity, uint64_t *nout, uint64_t *npath);
/* CondVarLenTraverse's DISTINCT endpoints of a bidirectional pattern (a)-[*min_hops..max_hops]-(b) with min_hops <= 1, from
 * each starts[i], over ntypes tensors' live layers: *reached is a new nstarts x n BOOL matrix whose row i holds every b the trail
 * DFS emits from starts[i] under B200_DIR_BOTH (B200_var_len_trails' endpoints, without multiplicity).  Over the undirected
 * multigraph G' with one edge per live relationship (a self-loop once): v != starts[i] is in row i iff dist_G'(s, v) <= max_hops;
 * starts[i] itself iff min_hops == 0 or G' holds a cycle through it of at most max_hops edges (a self-loop; two relationships to
 * one neighbour, in either direction or of different types; or a longer cycle).  max_hops = UINT64_MAX: unbounded.  Every type
 * needs mt.  Errors as B200_var_len_trails: NULL pointers or a NULL m / mt GrB_NULL_POINTER; ntypes outside 1 .. 65536
 * GrB_INVALID_VALUE; m / dp not UINT64 GrB_DOMAIN_MISMATCH; layers not square of one size GrB_DIMENSION_MISMATCH; a start >= n
 * GrB_INVALID_INDEX; host-resident layers, or min_hops > 1 (a walk is not a trail there: that pattern keeps the trail
 * enumerator), GrB_NOT_IMPLEMENTED; with no device GxB_GPU_ERROR before any host work.  nstarts == 0 or min_hops > max_hops:
 * empty rows, no device work.  No layer changes, apart from finishing pending tuples; no base is downloaded. */
GrB_Info B200_var_len_reach_both(GrB_Matrix *reached, const GrB_Index *starts, GrB_Index nstarts, const B200_TensorLayers *types,
                                 int ntypes, uint64_t min_hops, uint64_t max_hops);
/* allShortestPaths((a)-[:R1|R2*..max_hops]->(b)) for npairs bound pairs (AllShortestPathsOp::expand_row,
 * all_shortest_paths.rs:82-302): every shortest path from src[i] to dst[i] over ntypes tensors' live layers, in the reference's
 * emission order.  Adjacency is Graph::get_node_relationships_by_type's (see B200_var_len_trails); dir B200_DIR_OUT walks outgoing
 * edges (a right-to-left pattern still walks them from the arrow's source), B200_DIR_BOTH both halves.  min_hops is 1 (the
 * reference's planner rejects anything else); max_hops = UINT64_MAX: unbounded.  src[i] == dst[i] asks for the shortest cycles.
 * The order: a BFS from src in adjacency order records every entry into a node from the level before it (its predecessors, in
 * visit order); the paths are a DFS from dst that pushes a node's predecessors in list order, so the last one pops first.
 * Outputs, always written: out_count[i] (the number of shortest paths, saturating at UINT64_MAX; 0 = none), out_len[i] (edges
 * per path, 0 when none), out_p[npairs + 1] (paths written, a prefix over pairs) and *nedges (edges written).  path_edge NULL:
 * count only.  Otherwise pairs are filled in order, pair i from rank first[i] on (first NULL: 0), and filling stops at the first
 * path whose edges no longer fit edge_capacity; a caller drains a pair across calls with first[i] += paths written.  Path k's
 * edges are path_edge[E_k .. E_k + len), E_k = the edges of the paths before it, in src -> dst walk order, except for
 * src == dst, whose list starts with the closing edge (the reference keeps a cycle's predecessor-chain order); its nodes are
 * path_node[E_k + k .. E_k + k + len] following the edge list from src (at most 2 * edge_capacity entries).  A caller reverses
 * both lists for a right-to-left pattern.  Every type needs mt (the paths are recovered from dst over incoming edges).
 * Errors: NULL pointers or a NULL m / mt GrB_NULL_POINTER; ntypes outside 1 .. 65536 or dir not OUT / BOTH GrB_INVALID_VALUE;
 * m / dp not UINT64 GrB_DOMAIN_MISMATCH; layers not square of one size GrB_DIMENSION_MISMATCH; an endpoint >= n
 * GrB_INVALID_INDEX; host-resident layers GrB_NOT_IMPLEMENTED; with no device GxB_GPU_ERROR before any host work.  npairs == 0
 * or max_hops == 0: success with empty rows and no device work.  last_flops = the adjacency entries scanned.  No layer changes,
 * apart from finishing pending tuples; no base is downloaded.  Option "shortest_path_budget": candidates per piece of a forward
 * level (0: sized from free device memory). */
GrB_Info B200_all_shortest_paths(const GrB_Index *src, const GrB_Index *dst, GrB_Index npairs, const B200_TensorLayers *types,
                                 int ntypes, int dir, uint64_t max_hops, const uint64_t *first, uint64_t *out_count, uint32_t *out_len,
                                 uint64_t *out_p, uint64_t *path_edge, uint32_t *path_node, uint64_t edge_capacity, uint64_t *nedges);
/* Flags of the write plans below. */
#define B200_PLAN_COMMITTED 0x01 /* insert: m holds the pair, its value is to be reconciled (dm.erase) */
#define B200_PLAN_CANCEL 0x02    /* insert: COMMITTED and m's value equals the new inline value (dp.erase instead of dp.insert) */
#define B200_PLAN_MT_BASE 0x04   /* insert / remove: mt's base m holds (dst, src) */
#define B200_PLAN_EMPTIED 0x08   /* remove: the pair lost its last edge */
#define B200_PLAN_DEMOTED 0x10   /* remove: the pair is down to one edge, pr_val */
#define B200_PLAN_M_HAS 0x20     /* remove: m holds the pair */
#define B200_PLAN_M_EQ 0x40      /* remove: DEMOTED and m's value equals the survivor */
/* The read phase of Tensor::set_all_from_slices (tensor.rs:333-447) and of Tensor::remove_all's multi-edge path (:454-629) for a
 * whole batch, on the device, over one relationship type's layers as they stand before the batch (m, dp, dm, mt, me, and for
 * removes me_dp / me_dm; mt_dp / mt_dm are checked but not read).  The caller then makes the reference's write calls from the plan
 * and reads no layer.  No layer changes, apart from finishing pending tuples.
 * Insert: each distinct pair P with batch ids i1..ig in batch order; cur = dp's value if present, else none if dm holds P, else m's.
 *  - cur MULTI_EDGE: me entries i1..ig, no inline record;
 *  - cur a single id c: me entries c, i1..ig, inline MULTI_EDGE; COMMITTED when dp held P and m holds P;
 *  - none, g = 1: inline i1;  none, g >= 2: me entries i1..ig, inline MULTI_EDGE; COMMITTED when dm held P and m holds P.
 *  Inline records (in_src, in_dst, in_val, in_flags: COMMITTED, CANCEL, MT_BASE) at most n; me entries (me_key = src << 32 | dst,
 *  me_id, me_base = me's base m holds (key, id)) at most 2n.
 * Remove: each distinct pair with its distinct batch ids R, by Tensor::eff_get:
 *  - a single id x: an EMPTIED record when x is in R;
 *  - MULTI_EDGE with the merged id list L = (me \ me_dm) u me_dp, H = R n L nonempty, rem = L \ H: |rem| >= 2: me entries H; |rem|
 *    = 1: me entries L and a DEMOTED record, pr_val = the survivor; |rem| = 0: me entries L and an EMPTIED record.  A list of
 *    fewer than two ids (only reached by adding an id the pair already holds) takes the |rem| >= 2 row, as the host's walk does.
 *  Pair records (pr_*: EMPTIED / DEMOTED, M_HAS, MT_BASE, M_EQ; pr_val the survivor, else the pair's value before the batch) at most
 *  n; me entries at most 2n.  The reference lists emptied pairs in discovery order; its callers use them as a set.
 * Pairs ascending; a pair's me entries in the order above (insert) or ascending (remove).
 * Errors: m or mt NULL GrB_NULL_POINTER; m / dp not UINT64 GrB_DOMAIN_MISMATCH; layers not square of one size n
 * GrB_DIMENSION_MISMATCH; src / dst >= n or an id >= 2^60 GrB_INVALID_INDEX; host-resident m GrB_NOT_IMPLEMENTED; n == 0 success
 * with no device work; with no device GxB_GPU_ERROR before any host work. */
GrB_Info B200_Tensor_insert_plan(const B200_TensorLayers *t, const GrB_Index *srcs, const GrB_Index *dsts, const GrB_Index *ids,
                                 GrB_Index n, uint64_t *in_src, uint64_t *in_dst, uint64_t *in_val, uint8_t *in_flags, uint64_t *nin,
                                 uint64_t *me_key, uint64_t *me_id, uint8_t *me_base, uint64_t *nme);
GrB_Info B200_Tensor_remove_plan(const B200_TensorLayers *t, const GrB_Index *ids, const GrB_Index *srcs, const GrB_Index *dsts,
                                 GrB_Index n, uint64_t *pr_src, uint64_t *pr_dst, uint64_t *pr_val, uint8_t *pr_flags, uint64_t *npr,
                                 uint64_t *me_key, uint64_t *me_id, uint8_t *me_base, uint64_t *nme);
GrB_Info B200_sync(void);
GrB_Info B200_pool_trim(void); /* hand the caching allocator's free device blocks back to the driver */
void *B200_stream(void); /* the cudaStream_t every kernel of this library is launched on */
/* stats: "launches", "lib_launches", "last_flops", "total_flops", "last_path", "h2d_bytes", "d2h_bytes" */
uint64_t B200_get_stat(const char *name);
void B200_reset_stats(void);
/* with option "timing"=1 the library brackets its main kernels with CUDA events on its stream; this returns the
 * accumulated device time (ms), launch count and algorithmic bytes of one kernel family since the last reset:
 * "bits_pull", "bits_push", "heavy_accumulate", "bits_fill", "bits_count", "bits_delta", "bits_repair", the accumulating
 * products of union hops, "bits_pull_acc" and "bits_push_acc", "transpose", "bfs_expand", B200_bfs_delta's kernels over
 * dirty operands, "bfs_delta", B200_adjacency_delta's induced-layer kernels, "adj_build", B200_var_len_trails' kernels,
 * "var_len_trails", B200_var_len_reach_both's own kernels (its reach and closure levels count under the hop families),
 * "var_len_reach_both", B200_shortest_path's, "shortest_path", and B200_all_shortest_paths' (its adjacency fetches included),
 * "all_shortest_paths".  0 on success. */
int B200_kernel_stats(const char *name, double *ms, uint64_t *launches, uint64_t *bytes);
/* options: "bits_mode" (-1 auto,0 off,1 on), "pull_mode" (-1 auto,0 push,1 pull), "small_cap",
 * "bitmap_budget", "bits_min_flops", "timing" (0/1), "sync_after_op" (0/1) */
GrB_Info B200_set_option(const char *name, int64_t value);
const char *B200_last_error(void);
/* single-source BFS straight into caller buffers (int64 level/parent per vertex, -1 = unreached) */
GrB_Info B200_bfs(GrB_Matrix A, GrB_Index src, int64_t max_level, int64_t *level, int64_t *parent, int location,
                  uint64_t *edges_traversed);
/* what one BFS did: levels by direction, exchange volume / time of the partitioned form (device-event timed) */
typedef struct {
    uint64_t depth, edges, td_levels, bu_levels, sparse_levels, exchanges, exchanged_bytes;
    double device_ms, exchange_ms;
} B200_BfsInfo;
/* BFS with the `dest` early exit of LAGr_BreadthFirstSearch_Extended (lagraphx_bindings.rs:585-594; -1 = none).  Runs the
 * direction-optimising engine when the transpose mirror exists (B200_Matrix_prepare(A, 1)), else the top-down kernel. */
GrB_Info B200_bfs_ex(GrB_Matrix A, GrB_Index src, int64_t max_level, int64_t dest, int64_t *level, int64_t *parent, int location,
                     B200_BfsInfo *info);
/* B200_bfs_ex over relationship operands with pending writes (algo.BFS, algo_procedures.rs:1021-1166): the BFS walks
 * A = U_t (m[t] \ dm[t]) u dp[t], pattern only, with B200_reach_batch_delta's operand rules (m / dp may be UINT64; within a type
 * dp wins over dm; dm entries outside m have no effect; an entry one type holds survives another type's dm; dp / dm may be NULL
 * arrays or hold NULL entries).  level / parent / max_level / dest / location / info as for B200_bfs_ex (minimum-id parent).  The
 * direction-optimising engine runs on the operands in place: no union is built and no base is changed; each base's transpose
 * mirror is built on first use and cached on its handle, the deltas' transposes are built per call.  One operand without deltas
 * is exactly B200_Matrix_prepare(m[0], 1) + B200_bfs_ex.  Errors: nops < 1 GrB_INVALID_VALUE; operands not square of one size
 * GrB_DIMENSION_MISMATCH; host-resident operands GrB_NOT_IMPLEMENTED; src or dest >= n GrB_INVALID_INDEX; with no device
 * GxB_GPU_ERROR before any host work. */
GrB_Info B200_bfs_delta(const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops, GrB_Index src,
                        int64_t max_level, int64_t dest, int64_t *level, int64_t *parent, int location, B200_BfsInfo *info);
/* The shortestPath((a)-[:R1|R2*min_hops..max_hops]->(b)) expression for npairs bound pairs (ExprEval::eval_shortest_path,
 * eval.rs:1296-1513): the reference's bidirectional BFS, path for path.  The forward side walks the union of its nf operands
 * (fm, fdp, fdm) and the backward side that of its nb operands (bm, bdp, bdm), each with B200_reach_batch_delta's operand rules
 * (m / dp may be UINT64; within an operand dp wins over dm; an entry one operand holds survives another operand's dm; dp / dm may
 * be NULL arrays or hold NULL entries).  Each round expands the side with the smaller front (the forward one on a tie); a new
 * vertex's parent is its lowest-ranked front neighbour, the next front is ordered by (parent rank, vertex), and the meet is the
 * least (other side's depth, parent rank, vertex).  src == dst: the one-node path when min_hops == 0, else Null.
 * max_hops = UINT64_MAX: unbounded.  Row i is path_node[out_p[i] .. out_p[i+1]), from src[i] to dst[i]; an empty row is Null.
 * out_p (npairs + 1 entries) and *nnodes are always written; nodes only when they fit node_capacity, else GrB_INSUFFICIENT_SPACE
 * with *nnodes = the nodes needed.  The relationships between consecutive nodes are B200_expand_edges(DIR_BOTH, targets,
 * EDGES_FIRST)'s first entry per row.  Errors: nf or nb < 1, or min_hops > 1, GrB_INVALID_VALUE; operands not square of one size
 * GrB_DIMENSION_MISMATCH; an endpoint >= n GrB_INVALID_INDEX; host-resident operands GrB_NOT_IMPLEMENTED; with no device
 * GxB_GPU_ERROR before any host work.  npairs == 0: success with no device work.  last_flops = the neighbour entries scanned.
 * No layer changes, apart from finishing pending tuples; no base is downloaded.  Option "shortest_path_budget": neighbour entries
 * per piece of a round (0: sized from free device memory). */
GrB_Info B200_shortest_path(const GrB_Index *src, const GrB_Index *dst, GrB_Index npairs, const GrB_Matrix *fm, const GrB_Matrix *fdp,
                            const GrB_Matrix *fdm, int nf, const GrB_Matrix *bm, const GrB_Matrix *bdp, const GrB_Matrix *bdm, int nb,
                            uint64_t min_hops, uint64_t max_hops, uint64_t *out_p, uint32_t *path_node, uint64_t node_capacity,
                            uint64_t *nnodes);
/* The adjacency the algorithm procedures run on (algo.pageRank / algo.WCC / algo.labelPropagation, algo_procedures.rs:718-732,
 * 816-832, 1207-1223), built on the device in one call over relationship operands with pending writes.  *A is a new BOOL, iso
 * matrix: the union over t of the induced effective layer (m[t] \ dm[t]) u dp[t], restricted to the kept vertices (rows and
 * columns) with both indices replaced by their rank among them.
 *   keep == NULL: the vertices below n_out, A is n_out x n_out (the reference's dup + resize to node_count + deleted_nodes_count:
 *                 entries at or beyond n_out are dropped, rows beyond ncols(m) are empty).  n_out must be below 2^32.
 *   keep != NULL: keep[0 .. nkeep) strictly ascending ids below ncols(m[0]), A is nkeep x nkeep and vertex keep[k] is index k
 *                 (the compact matrix of a label filter).  nkeep == 0 gives a 0 x 0 matrix.
 *   symmetric:    A u A' (build_symmetric_adjacency_matrix, the input of WCC and CDLP).
 * Only the kept rows of each m, dp and dm are read.  Operand rules as B200_reach_batch_delta (m / dp may be UINT64, values are
 * ignored; within a type dp wins over dm; dm entries outside m have no effect; an entry one type holds survives another type's dm;
 * dp / dm may be NULL arrays or hold NULL entries).  No operand is changed.  Errors: nops < 1 or n_out >= 2^32 GrB_INVALID_VALUE;
 * operands not square of one size GrB_DIMENSION_MISMATCH; keep not strictly ascending or holding an id >= ncols(m[0])
 * GrB_INVALID_INDEX; host-resident operands GrB_NOT_IMPLEMENTED; with no device GxB_GPU_ERROR before any host work. */
GrB_Info B200_adjacency_delta(GrB_Matrix *A, const GrB_Matrix *m, const GrB_Matrix *dp, const GrB_Matrix *dm, int nops,
                              GrB_Index n_out, const GrB_Index *keep, GrB_Index nkeep, int symmetric);
/* 1-D row-block partitioned BFS over NCCL (BASELINE config 5; SURVEY 8e).  Rank 0 obtains the 128-byte id, the caller ships it
 * to the other ranks, every rank calls B200_comm_init; world == 1 needs no id.  NCCL is resolved with dlopen at run time. */
typedef struct B200_Comm_opaque *B200_Comm;
GrB_Info B200_comm_unique_id(uint8_t *id128);
GrB_Info B200_comm_init(B200_Comm *comm, int rank, int world, const uint8_t *id128);
GrB_Info B200_comm_free(B200_Comm *comm);
/* Alocal / ATlocal: rows [row_lo, row_lo + nloc) of the n x n adjacency matrix and of its transpose (global column ids); blocks
 * are ceil(n / world) rounded up to a multiple of 64.  level_local / parent_local: int64[nloc].  Collective over `comm`. */
GrB_Info B200_bfs_partitioned(GrB_Matrix Alocal, GrB_Matrix ATlocal, uint64_t n, uint64_t row_lo, B200_Comm comm, GrB_Index src,
                              int64_t max_level, int64_t dest, int64_t *level_local, int64_t *parent_local, int location,
                              B200_BfsInfo *info);

#ifdef __cplusplus
}
#endif
#endif /* B200GRB_H */
