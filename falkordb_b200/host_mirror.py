"""ctypes binding of libfdbhost.so, the C++ host mirror of the reference's Tensor and CondTraverse (csrc/host): a relationship
Tensor built by GRAPH.BULK's device-side load and changed by batched writes that stay pending (through the reference's read phase
or the device plans, B200_Tensor_insert_plan / B200_Tensor_remove_plan), and the routes that read its
relationship ids (B200_expand_edges, Tensor::get per pair, bind_edge's traversal-then-get), CondVarLenTraverse's trails
(B200_var_len_trails, or the reference's DFS) and its bidirectional DISTINCT endpoints (B200_var_len_reach_both), the shortestPath
expression (B200_shortest_path, or the reference's NeighborIter BFS), allShortestPaths (B200_all_shortest_paths, or
the reference's expand_row), and the algo.BFS, algo.pageRank, algo.WCC
and algo.labelPropagation procedures over them."""
import ctypes as C
import os

import numpy as np

from ._lib import U64

_HERE = os.path.dirname(os.path.abspath(__file__))
_L = None

ROUTE_DEVICE, ROUTE_BY_GET, ROUTE_TRAVERSE_GET = 0, 1, 2
BFS_DEVICE, BFS_BY_EXTRACT = 0, 1
SP_DEVICE, SP_BY_ITER = 0, 1
ASP_DEVICE, ASP_BY_ITER = 0, 1
ALGO_DEVICE, ALGO_BY_EXTRACT = 0, 1
WRITE_REFERENCE, WRITE_DEVICE = 0, 1


def host():
    global _L
    if _L is not None:
        return _L
    L = C.CDLL(os.path.join(_HERE, "libfdbhost.so"))
    P = C.c_void_p
    L.fdbh_tensor_bulk_load.argtypes = [U64, P, P, P, U64]
    L.fdbh_tensor_bulk_load.restype = P
    L.fdbh_tensor_free.argtypes = [P]
    L.fdbh_tensor_set_all.argtypes = [P, P, P, P, U64]
    L.fdbh_tensor_remove_all.argtypes = [P, P, P, P, U64]
    L.fdbh_tensor_layers.argtypes = [P, P]
    L.fdbh_tensor_set_all_dev.argtypes = [P, P, P, P, U64]
    L.fdbh_tensor_remove_all_dev.argtypes = [P, P, P, P, U64, C.POINTER(P), C.POINTER(P), C.POINTER(U64)]
    L.fdbh_tensor_remove_all_emptied.argtypes = [P, P, P, P, U64, C.POINTER(P), C.POINTER(P), C.POINTER(U64)]
    L.fdbh_tensor_counts.argtypes = [P, P]
    L.fdbh_tensor_dup.argtypes = [P]
    L.fdbh_tensor_dup.restype = P
    L.fdbh_tensor_fold_oversized.argtypes = [P]
    L.fdbh_tensor_flush.argtypes = [P]
    L.fdbh_tensor_edge_count.argtypes = [P]
    L.fdbh_tensor_edge_count.restype = C.c_int64
    L.fdbh_vm_set_all.argtypes = [P, P, P, U64, C.c_int, C.c_int]
    L.fdbh_vm_state.argtypes = [P, P, P]
    L.fdbh_run_write_test.argtypes = [C.c_char_p, C.c_int]
    L.fdbh_expand_edges.argtypes = [P, U64, P, P, U64, C.c_int, C.c_int, C.c_int] + [P] * 5 + [C.POINTER(U64)]
    vl = [P, U64, C.c_int, P, P, U64, U64, U64, P, U64, C.c_int]
    L.fdbh_var_len_trails.argtypes = vl + [U64] + [P] * 5 + [C.POINTER(U64)] * 2
    L.fdbh_var_len_trails_dfs.argtypes = vl + [P] * 5 + [C.POINTER(U64)] * 2
    L.fdbh_var_len_reach_both.argtypes = [P, U64, P, U64, U64, U64, C.POINTER(P), C.POINTER(P), C.POINTER(U64)]
    L.fdbh_shortest_path.argtypes = [P, P, U64, P, U64, C.c_int, U64, U64, P, P, U64, C.c_int] + [C.POINTER(P)] * 4
    L.fdbh_all_shortest_paths.argtypes = [P, U64, P, U64, C.c_int, U64, P, P, U64, C.c_int, U64] + [C.POINTER(P)] * 5
    L.fdbh_algo_bfs.argtypes = [P, P, U64, P, U64, P, U64, U64, C.c_int64, C.c_int, C.c_int, P, C.POINTER(U64), P, C.POINTER(U64)]
    algo = [P, P, U64, P, U64, P, U64, U64, P, U64]
    L.fdbh_algo_pagerank.argtypes = algo + [C.c_int, P, P, C.POINTER(U64)]
    L.fdbh_algo_wcc.argtypes = algo + [C.c_int, P, P, C.POINTER(U64)]
    L.fdbh_algo_cdlp.argtypes = algo + [C.c_int, C.c_int, P, P, C.POINTER(U64)]
    L.fdbh_vm_new.argtypes = [U64, U64]
    L.fdbh_vm_new.restype = P
    L.fdbh_vm_free.argtypes = [P]
    L.fdbh_vm_set.argtypes = [P, U64, U64]
    L.fdbh_vm_remove.argtypes = [P, U64, U64]
    L.fdbh_free.argtypes = [P]
    L.fdbh_last_message.restype = C.c_char_p
    _L = L
    return L


def _u64(*xs):
    return [np.ascontiguousarray(x, dtype=np.uint64) for x in xs]


class Tensor:
    """csrc/host/tensor.hpp's Tensor over n vertices, loaded with the edges (src[k], dst[k], ids[k]) by Tensor::bulk_load"""

    def __init__(self, n, src, dst, ids):
        self.L = host()
        a = _u64(src, dst, ids)
        self.h = self.L.fdbh_tensor_bulk_load(n, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, len(a[0]))
        if not self.h:
            raise RuntimeError(self.L.fdbh_last_message().decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.L.fdbh_tensor_free(self.h)
            self.h = None

    @classmethod
    def _adopt(cls, h):
        t = cls.__new__(cls)
        t.L = host()
        if not h:
            raise RuntimeError(t.L.fdbh_last_message().decode())
        t.h = h
        return t

    def _check(self, rc):
        if rc:
            raise RuntimeError(self.L.fdbh_last_message().decode())

    def add(self, src, dst, ids, route=WRITE_REFERENCE):
        """Tensor::set_all_from_slices, or with route=WRITE_DEVICE set_all_from_slices_dev (its read phase as one device plan)"""
        a = _u64(src, dst, ids)
        fn = self.L.fdbh_tensor_set_all_dev if route == WRITE_DEVICE else self.L.fdbh_tensor_set_all
        self._check(fn(self.h, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, len(a[0])))

    def remove(self, ids, src, dst, route=WRITE_REFERENCE):
        """Tensor::remove_all, or with route=WRITE_DEVICE remove_all_dev.  Returns the emptied pairs as a (k, 2) uint64 array: the
        reference lists them in discovery order, the device route ascending."""
        a = _u64(ids, src, dst)
        fn = self.L.fdbh_tensor_remove_all_dev if route == WRITE_DEVICE else self.L.fdbh_tensor_remove_all_emptied
        ps, pd, nv = C.c_void_p(), C.c_void_p(), U64(0)
        self._check(fn(self.h, a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, len(a[0]), C.byref(ps), C.byref(pd), C.byref(nv)))
        k = nv.value
        out = np.zeros((k, 2), np.uint64)
        for col, x in enumerate((ps, pd)):
            if k:
                out[:, col] = np.frombuffer((C.c_char * (8 * k)).from_address(x.value), np.uint64)
            self.L.fdbh_free(x)
        return out

    def dup(self):
        """Tensor::dup: a new version sharing the layers copy-on-write"""
        return Tensor._adopt(self.L.fdbh_tensor_dup(self.h))

    def fold_oversized(self):
        self._check(self.L.fdbh_tensor_fold_oversized(self.h))

    def flush(self):
        self._check(self.L.fdbh_tensor_flush(self.h))

    def edge_count(self):
        n = self.L.fdbh_tensor_edge_count(self.h)
        if n < 0:
            raise RuntimeError(self.L.fdbh_last_message().decode())
        return n

    def counts(self):
        """the six Delta counters: dp, dm, mt's dp, dm, me's dp, dm"""
        out = np.zeros(6, np.uint64)
        self._check(self.L.fdbh_tensor_counts(self.h, out.ctypes.data))
        return out

    def tuples(self):
        """the nine layers' stored entries (TENSOR_LAYERS order) as (rows, cols, values or None) numpy arrays, after Tensor::wait()"""
        return [_tuples(h, k < 2) for k, h in enumerate(self.layers())]

    def layers(self):
        """the nine layer handles in B200_TensorLayers order, after Tensor::wait(); valid until the tensor changes"""
        out = (C.c_void_p * 9)()
        if self.L.fdbh_tensor_layers(self.h, out):
            raise RuntimeError(self.L.fdbh_last_message().decode())
        return [out[k] for k in range(9)]


def expand_edges(tensors, sources, dir, mode, targets=None, route=ROUTE_BY_GET):
    """fdbh_expand_edges over Tensor objects: (p, node, edge, type, rev) as numpy arrays"""
    L = host()
    (src,) = _u64(sources)
    tg = None if targets is None else _u64(targets)[0]
    ts = (C.c_void_p * len(tensors))(*[t.h for t in tensors])
    ptrs = [C.c_void_p() for _ in range(5)]
    nv = U64(0)
    rc = L.fdbh_expand_edges(ts, len(tensors), src.ctypes.data, None if tg is None else tg.ctypes.data, len(src), dir, mode, route,
                             *[C.byref(x) for x in ptrs], C.byref(nv))
    if rc:
        raise RuntimeError(L.fdbh_last_message().decode())
    m = nv.value
    out = []
    for x, dt, k in zip(ptrs, (np.uint64, np.uint32, np.uint64, np.uint16, np.uint8), (len(src) + 1, m, m, m, m)):
        nbytes = k * np.dtype(dt).itemsize
        out.append(np.frombuffer((C.c_char * nbytes).from_address(x.value), dt).copy() if k else np.zeros(0, dt))
        L.fdbh_free(x)
    return tuple(out)


def var_len_trails(tensors, starts, dir, min_hops=1, max_hops=None, dests=None, labels=(), emit_path=True, route=ROUTE_DEVICE,
                   tree_capacity=None):
    """CondVarLenTraverse's trails over Tensor objects: route ROUTE_DEVICE (fdbh_var_len_trails, one B200_var_len_trails call) or
    ROUTE_BY_GET (fdbh_var_len_trails_dfs, the reference's DFS over TypesAdjacency).  labels: VersionedMatrix objects, None for a
    label the graph lacks.  Returns a dict of numpy uint64 arrays: p, end, hops, and with emit_path edges and nodes in walk order."""
    L = host()
    (src,) = _u64(starts)
    ds = None if dests is None else np.ascontiguousarray(dests, dtype=np.int64)
    ts = (C.c_void_p * max(1, len(tensors)))(*[t.h for t in tensors])
    lb = (C.c_void_p * max(1, len(labels)))(*[None if x is None else x.h for x in labels])
    mx = (1 << 64) - 1 if max_hops is None else int(max_hops)
    ptrs = [C.c_void_p() for _ in range(5)]
    nv, npth = U64(0), U64(0)
    args = [ts, len(tensors), dir, src.ctypes.data, None if ds is None else ds.ctypes.data, len(src), int(min_hops), mx, lb, len(labels),
            1 if emit_path else 0]
    if route == ROUTE_DEVICE:
        rc = L.fdbh_var_len_trails(*args, (1 << 64) - 1 if tree_capacity is None else int(tree_capacity), *[C.byref(x) for x in ptrs],
                                   C.byref(nv), C.byref(npth))
    else:
        rc = L.fdbh_var_len_trails_dfs(*args, *[C.byref(x) for x in ptrs], C.byref(nv), C.byref(npth))
    if rc:
        raise RuntimeError(L.fdbh_last_message().decode())
    m, q = nv.value, npth.value
    out = {}
    for name, x, k in zip(("p", "end", "hops", "edges", "nodes"), ptrs, (len(src) + 1, m, m, q, q + m if emit_path else 0)):
        out[name] = np.frombuffer((C.c_char * (8 * k)).from_address(x.value), np.uint64).copy() if k else np.zeros(0, np.uint64)
        L.fdbh_free(x)
    return out


def var_len_reach_both(tensors, starts, min_hops=1, max_hops=None):
    """CondVarLenTraverse's bidirectional fast path over Tensor objects (fdbh_var_len_reach_both, one B200_var_len_reach_both
    call): the DISTINCT (row, node) pairs as a (k, 2) uint64 array in row order"""
    L = host()
    (src,) = _u64(starts)
    ts = (C.c_void_p * max(1, len(tensors)))(*[t.h for t in tensors])
    pr, pn, nv = C.c_void_p(), C.c_void_p(), U64(0)
    if L.fdbh_var_len_reach_both(ts, len(tensors), src.ctypes.data, len(src), int(min_hops), (1 << 64) - 1 if max_hops is None else int(max_hops),
                                 C.byref(pr), C.byref(pn), C.byref(nv)):
        raise RuntimeError(L.fdbh_last_message().decode())
    k = nv.value
    out = np.zeros((k, 2), np.uint64)
    for col, x in enumerate((pr, pn)):
        if k:
            out[:, col] = np.frombuffer((C.c_char * (8 * k)).from_address(x.value), np.uint64)
        L.fdbh_free(x)
    return out


class VersionedMatrix:
    """csrc/host/versioned_matrix.hpp's VersionedMatrix<bool> (the graph's adjacency matrix): set / remove stay pending"""

    def __init__(self, n):
        self.L = host()
        self.h = self.L.fdbh_vm_new(n, n)
        if not self.h:
            raise RuntimeError(self.L.fdbh_last_message().decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.L.fdbh_vm_free(self.h)
            self.h = None

    def set(self, i, j):
        if self.L.fdbh_vm_set(self.h, int(i), int(j)):
            raise RuntimeError(self.L.fdbh_last_message().decode())

    def remove(self, i, j):
        if self.L.fdbh_vm_remove(self.h, int(i), int(j)):
            raise RuntimeError(self.L.fdbh_last_message().decode())

    def set_all(self, rows, cols, new=False, route=WRITE_REFERENCE):
        """VersionedMatrix::set_all<NEW>, or with route=WRITE_DEVICE set_all_dev<NEW> (one batched base probe)"""
        r, c = _u64(rows, cols)
        if self.L.fdbh_vm_set_all(self.h, r.ctypes.data, c.ctypes.data, len(r), 1 if new else 0, route):
            raise RuntimeError(self.L.fdbh_last_message().decode())

    def state(self):
        """(the two Delta counters, the (rows, cols) of m, dp and dm)"""
        cnt, hs = np.zeros(2, np.uint64), (C.c_void_p * 3)()
        if self.L.fdbh_vm_state(self.h, cnt.ctypes.data, hs):
            raise RuntimeError(self.L.fdbh_last_message().decode())
        return cnt, [_tuples(hs[k], False)[:2] for k in range(3)]


def _tuples(h, valued):
    from ._lib import lib, check
    L = lib()
    n = U64(0)
    check(L.GrB_Matrix_nvals(C.byref(n), h))
    k = n.value
    rows, cols = np.zeros(max(k, 1), np.uint64), np.zeros(max(k, 1), np.uint64)
    vals = np.zeros(max(k, 1), np.uint64) if valued else None
    nv = U64(max(k, 1))
    fn = L.GrB_Matrix_extractTuples_UINT64 if valued else L.GrB_Matrix_extractTuples_BOOL
    check(fn(rows.ctypes.data, cols.ctypes.data, None if vals is None else vals.ctypes.data, C.byref(nv), h))
    return rows[:k], cols[:k], None if vals is None else vals[:k]


def run_write_test(name, route):
    """one transcribed tensor.rs test with its writes through `route` (WRITE_REFERENCE / WRITE_DEVICE); '' on success"""
    L = host()
    rc = L.fdbh_run_write_test(name.encode(), route)
    return "" if rc == 0 else L.fdbh_last_message().decode()


def algo_bfs(adj, all_types, named, src, max_depth=-1, want_edges=True, deleted=(), route=BFS_DEVICE):
    """fdbh_algo_bfs: algo.BFS from `src` over `named` Tensors, or over the adjacency VersionedMatrix `adj` when none is named;
    relationship ids from `named`, or from `all_types` when none is named.  Returns (nodes, edges) as uint64 arrays."""
    L = host()
    (dl,) = _u64(sorted(deleted))
    at = (C.c_void_p * max(1, len(all_types)))(*[t.h for t in all_types])
    nt = (C.c_void_p * max(1, len(named)))(*[t.h for t in named])
    ptrs = [C.c_void_p(), C.c_void_p()]
    nn, ne = U64(0), U64(0)
    rc = L.fdbh_algo_bfs(None if adj is None else adj.h, at, len(all_types), nt, len(named), dl.ctypes.data, len(dl), int(src),
                         int(max_depth), 1 if want_edges else 0, route, C.byref(ptrs[0]), C.byref(nn), C.byref(ptrs[1]), C.byref(ne))
    if rc:
        raise RuntimeError(L.fdbh_last_message().decode())
    out = []
    for x, k in zip(ptrs, (nn.value, ne.value)):
        out.append(np.frombuffer((C.c_char * (8 * k)).from_address(x.value), np.uint64).copy() if k else np.zeros(0, np.uint64))
        L.fdbh_free(x)
    return tuple(out)


def shortest_path(adj, all_types, named, srcs, dsts, directed=True, min_hops=1, max_hops=None, route=SP_DEVICE):
    """fdbh_shortest_path: shortestPath((a)-[:named*min_hops..max_hops]->(b)) per pair (srcs[i], dsts[i]) over `named` Tensors (None
    entries: types the graph lacks), or over the adjacency VersionedMatrix `adj` when none is named; relationship ids from `named`,
    or from `all_types` when none is named.  Returns one entry per pair: (nodes, ids) as lists, or None (Null)."""
    L = host()
    s, d = _u64(srcs, dsts)
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    named = list(named or ())
    ptrs = [C.c_void_p() for _ in range(4)]
    rc = L.fdbh_shortest_path(None if adj is None else adj.h, arr(all_types), len(all_types), arr(named), len(named), 1 if directed else 0,
                              int(min_hops), (1 << 64) - 1 if max_hops is None else int(max_hops), s.ctypes.data, d.ctypes.data, len(s),
                              route, *[C.byref(x) for x in ptrs])
    if rc:
        raise RuntimeError(L.fdbh_last_message().decode())
    n = len(s)
    p = np.frombuffer((C.c_char * (8 * (n + 1))).from_address(ptrs[0].value), np.uint64).copy()
    ep = np.frombuffer((C.c_char * (8 * (n + 1))).from_address(ptrs[2].value), np.uint64).copy()
    nodes = np.frombuffer((C.c_char * (8 * int(p[-1]))).from_address(ptrs[1].value), np.uint64).tolist() if p[-1] else []
    ids = np.frombuffer((C.c_char * (8 * int(ep[-1]))).from_address(ptrs[3].value), np.uint64).tolist() if ep[-1] else []
    for x in ptrs:
        L.fdbh_free(x)
    return [(nodes[p[i]:p[i + 1]], ids[ep[i]:ep[i + 1]]) if p[i + 1] > p[i] else None for i in range(n)]


def all_shortest_paths(all_types, named, srcs, dsts, directed=True, max_hops=None, route=ASP_DEVICE, window=1 << 22):
    """fdbh_all_shortest_paths: allShortestPaths((a)-[:named*..max_hops]->(b)) per pair (srcs[i], dsts[i]) over `named` Tensors (None
    entries: types the graph lacks), or over `all_types` when none is named; directed False: both directions.  route ASP_DEVICE
    drains B200_all_shortest_paths in windows of at most `window` edges.  Returns one list per pair of its paths, in the
    reference's emission order, each (edges, nodes) as lists."""
    L = host()
    s, d = _u64(srcs, dsts)
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    named = list(named or ())
    ptrs = [C.c_void_p() for _ in range(5)]
    rc = L.fdbh_all_shortest_paths(arr(all_types), len(all_types), arr(named), len(named), 1 if directed else 0,
                                   (1 << 64) - 1 if max_hops is None else int(max_hops), s.ctypes.data, d.ctypes.data, len(s), route,
                                   int(window), *[C.byref(x) for x in ptrs])
    if rc:
        raise RuntimeError(L.fdbh_last_message().decode())
    n = len(s)
    get = lambda k, m: np.frombuffer((C.c_char * (8 * m)).from_address(ptrs[k].value), np.uint64).tolist() if m else []
    pp, count, ln = get(0, n + 1), get(1, n), get(2, n)
    ne = sum(c * l for c, l in zip(count, ln))
    edges, nodes = get(3, ne), get(4, ne + pp[-1])
    for x in ptrs:
        L.fdbh_free(x)
    out, e = [], 0
    for i in range(n):
        paths = []
        for _ in range(count[i]):
            k = len(paths) + pp[i]
            paths.append((edges[e:e + ln[i]], nodes[e + k:e + k + ln[i] + 1]))
            e += ln[i]
        out.append(paths)
    return out


def _algo(fn, dt, adj, all_types, named, labels, node_count, deleted, route, *extra):
    L = host()
    (dl,) = _u64(sorted(deleted))
    arr = lambda xs: (C.c_void_p * max(1, len(xs)))(*[None if x is None else x.h for x in xs])
    named, labels = list(named or ()), list(labels or ())
    ptrs = [C.c_void_p(), C.c_void_p()]
    nv = U64(0)
    rc = getattr(L, fn)(None if adj is None else adj.h, arr(all_types), len(all_types), arr(named), len(named), arr(labels), len(labels),
                        int(node_count), dl.ctypes.data, len(dl), *extra, route, C.byref(ptrs[0]), C.byref(ptrs[1]), C.byref(nv))
    if rc:
        raise RuntimeError(L.fdbh_last_message().decode())
    out = []
    for x, t in zip(ptrs, (np.uint64, dt)):
        k = nv.value
        out.append(np.frombuffer((C.c_char * (8 * k)).from_address(x.value), t).copy() if k else np.zeros(0, t))
        L.fdbh_free(x)
    return tuple(out)


def algo_pagerank(adj, all_types, named=(), labels=(), node_count=0, deleted=(), route=ALGO_DEVICE):
    """fdbh_algo_pagerank: algo.pageRank over the adjacency VersionedMatrix `adj`, or over the `named` Tensors (None: a type the
    graph does not have); `labels`: () or one label VersionedMatrix (None: a missing label); `node_count` live nodes, `deleted` the
    deleted ids.  Returns (nodes uint64, scores float64)."""
    return _algo("fdbh_algo_pagerank", np.float64, adj, all_types, named, labels, node_count, deleted, route)


def algo_wcc(adj, all_types, named=(), labels=(), node_count=0, deleted=(), route=ALGO_DEVICE):
    """fdbh_algo_wcc: algo.WCC, arguments as algo_pagerank with any number of labels (nodeLabels).  Returns (nodes uint64,
    component ids int64): the component ids are compact indices, as the procedure returns them."""
    return _algo("fdbh_algo_wcc", np.int64, adj, all_types, named, labels, node_count, deleted, route)


def algo_cdlp(adj, all_types, named=(), labels=(), node_count=0, deleted=(), max_iterations=10, route=ALGO_DEVICE):
    """fdbh_algo_cdlp: algo.labelPropagation, arguments as algo_wcc.  Returns (nodes uint64, community ids int64)."""
    return _algo("fdbh_algo_cdlp", np.int64, adj, all_types, named, labels, node_count, deleted, route, int(max_iterations))
