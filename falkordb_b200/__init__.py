"""falkordb_b200 -- H100-native (sm_90a) GraphBLAS traversal backend behind FalkorDB's graph store.

The product is the C-ABI shared library ``libb200grb.so`` (include/b200grb.h); this package is the
thin host-side mirror of the reference's GraphBLAS wrapper (graph/src/graph/graphblas/matrix.rs)
used by the tests and the benchmark.  There is no CPU fallback: importing works without a GPU
(so the symbol table can be checked), every bulk call fails loudly without one.
"""
from ._lib import lib, GrbError, check, LIB_PATH, INFO  # noqa: F401
from .grb import Matrix, Descriptor, init, rmat, get_stat, reset_stats, set_option, sync, bfs, wait_ticket, traverse_to_host, traverse_batch, multi_source_reach, reach_batch, adjacency, OUT_AUTO, OUT_BITMAP, OUT_CSR, expand_edges, DIR_OUT, DIR_IN, DIR_BOTH, EDGES_ALL, EDGES_FIRST, insert_plan, remove_plan, var_len_trails, var_len_reach_both, shortest_path, all_shortest_paths  # noqa: F401
