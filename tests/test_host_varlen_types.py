"""CondVarLenTraverse's trail enumerator over several relationship types with destination labels (TypesAdjacencyT in
falkordb_b200/csrc/host/cond_var_len_traverse.hpp) against a brute-force enumeration of every trail: parallel edges on one pair in
two types and inside one type, self-loops, a cycle, Out / In / Both, fixed destinations, and labels present, absent or missing.
The DFS makes no GraphBLAS call here, so this runs without a GPU."""
from test_host_tensor import run


def test_var_len_trails_over_types_with_labels_host_only():
    run("var_len_types_labels_logic")
