// frontier.cuh -- what the sources of the frontier bit-matrix path share (bits.cu: the frontier's form; csr_push.cu: the push
// straight from a CSR frontier and the delta terms; bits_hop.cu: the bit-matrix hop and the exact dirty-hop repair).
//
// FalkorDB's CondTraverse drives GrB_mxm with a short-fat left operand: F is |batch| x n with
// |batch| <= 1024 rows (graph/src/runtime/batch.rs:81, runtime/ops/cond_traverse.rs:600-605).
// For such operands the row-wise product F*A is the multi-source frontier expansion
//        Y[j] |= X[k]   for every edge (k,j) of A,    X[k] = bitmask of the F rows holding k,
// i.e. ONE pass over A serves up to 64*W frontier rows at once.  F lives as a vertex-major
// bit-matrix (DevBits) between hops; the sorted CSR the reference iterates
// (matrix.rs:1471-1605) is materialised only when something observes it.
//   push : active vertices only, load-balanced flat expansion, RED.OR.64 into Y
//   pull : stream A' (CSC of A) row by row, gather X[k], plain stores -- no atomics
// Algorithmic bytes per hop (pull): 4*nnz(A') + 8*(n+1) + 8*W*nnz(A') gathers (L2) + 8*W*n.
#pragma once
#include "common.cuh"
#include "ops.cuh"
#include <cub/block/block_reduce.cuh>
#include <string>
#include <type_traits>

namespace b200 {

// how the lanes of a warp share a W-word vertex record: a lane moves at most 16 bytes per instruction on sm_90 (LDG.128 / STG.128)
__host__ __device__ constexpr int pull_split(int W) { return W >= 2 ? W / 2 : 1; }
template <int W> struct PullCfg {
    static constexpr int SPLIT = pull_split(W);    // lanes per vertex record
    static constexpr int WL = W / SPLIT;           // words per lane
    static constexpr int VG = 8 / SPLIT;           // vertices gathered per 8-lane group and unroll step
};
static const u64 PUSH_CHUNK = 8192;

template <int WL> __device__ __forceinline__ void ld_part(u64 (&x)[WL], const u64 *p) {
    static_assert(WL == 1 || WL == 2, "a record part is one 8- or 16-byte load");
    if constexpr (WL == 1) { x[0] = __ldg(p); }
    else { ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2 *>(p)); x[0] = v.x; x[1] = v.y; }
}

inline void require_natural(const DevBits &X, const char *what) {
    if (X.permuted()) throw GrbError(-101, std::string(what) + ": frontier is in permuted form (internal error: bits_naturalise was not called)");
}
// accumulate mode (union hops): the product is ORed into Y, which must already hold a natural-order product of the same shape
inline void require_acc_target(const DevBits &Y, u64 nrows, u64 ncols, u32 W) {
    require_natural(Y, "accumulating product");
    if (Y.nrows != nrows || Y.ncols != ncols || Y.W != W) throw GrbError(-6, "accumulating product: target shape differs");
}
// vertex -> position of the order X is stored in (null: natural order), for the passes that address single vertices in place
inline const u32 *pos_table(const DevBits &X) { return X.permuted() ? X.pperm->ptr : nullptr; }
inline void require_pos_table(const DevBits &X, const char *what) {
    if (X.permuted() && !X.pperm) throw GrbError(-101, std::string(what) + ": permuted frontier without its vertex -> position table");
}

// f(std::integral_constant<int, W>{}) for the word counts a frontier can have (bits_words_for)
template <class F> auto with_words(u32 W, F &&f) {
    switch (W) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    default: throw GrbError(-8, "bit-frontier: unsupported word count");
    }
}

} // namespace b200
