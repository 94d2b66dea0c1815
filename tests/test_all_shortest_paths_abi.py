"""allShortestPaths without a GPU: a Python transcription of the reference's AllShortestPathsOp::expand_row (all_shortest_paths.rs:
128-302), held to the reference flow test's graphs and expectations (a golden file); the level-synchronous statement that
all_shortest_paths.cu implements (forward ranks in pieces, backward predecessors from the reverse adjacency, saturating counts,
unranking, output windows) held equal to the transcription, path for path and in order, on 1,200 random multigraphs; unranking
at saturated counts; and B200_all_shortest_paths' argument errors, empty calls, and
GxB_GPU_ERROR without a device."""
import ctypes as C
import json
import os
from collections import deque

import numpy as np
import pytest

import falkordb_b200 as fb
from falkordb_b200 import host_mirror as hm
from falkordb_b200._lib import lib, U64
from falkordb_b200.grb import Matrix, _layers

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "all_shortest_paths_flow_cases.json")
INF = None
SAT = (1 << 64) - 1


def _has_gpu():
    import torch
    return torch.cuda.is_available()


class Graph:
    """effective relationships {type: [(u, v, id)]} and the pattern's types in order; adjacency in get_node_relationships_by_type's
    order (per type the outgoing half by (neighbour, id), then the incoming half by (source, id), a self-loop once under Both)"""

    def __init__(self, rels, order):
        self.rels, self.order = rels, [t for t in order if t in rels]
        self._fwd, self._rev = {}, {}

    def adj(self, node, both):
        k = (node, both)
        if k not in self._fwd:
            out = []
            for t in self.order:
                r = self.rels[t]
                out += sorted([e for e in r if e[0] == node], key=lambda e: (e[1], e[2]))
                if both:
                    out += sorted([e for e in r if e[1] == node and e[0] != node], key=lambda e: (e[0], e[2]))
            self._fwd[k] = out
        return self._fwd[k]

    def rev(self, v, both):
        """the reverse adjacency the backward phase fetches: (u, id, type index, half as u sees it), in the fetch's order (incoming
        edges for Out; both halves of v for Both)"""
        k = (v, both)
        if k not in self._rev:
            out = []
            for ti, t in enumerate(self.order):
                r = self.rels[t]
                if both:
                    out += [(e[1], e[2], ti, 0 if e[1] == v else 1) for e in sorted([e for e in r if e[0] == v], key=lambda e: (e[1], e[2]))]
                out += [(e[0], e[2], ti, 0) for e in sorted([e for e in r if e[1] == v and (not both or e[0] != v)], key=lambda e: (e[0], e[2]))]
            self._rev[k] = out
        return self._rev[k]


def expand_row(g, both, max_hops, src, dst):
    """the transcription: BFS then the DFS backtrack; [(edges, nodes)] in emission order (edges src -> dst, a cycle's from its
    closing edge; nodes following the edges from src)"""
    max_hops = (1 << 64) if max_hops is None else max_hops
    preds, dist, queue = {}, {src: 0}, deque([src])
    is_cycle, sd = src == dst, None
    while queue:
        cur = queue.popleft()
        d = dist[cur]
        if sd is not None and d >= sd:
            continue
        if d >= max_hops:
            continue
        for es, ed, eid in g.adj(cur, both):
            if es == cur:
                nxt = ed
            elif both and ed == cur and es != cur:
                nxt = es
            else:
                continue
            nd = d + 1
            if is_cycle and nxt == src:
                if sd is None:
                    sd = nd
                    preds.setdefault(nxt, []).append((cur, eid))
                elif nd == sd:
                    preds.setdefault(nxt, []).append((cur, eid))
                continue
            if nxt in dist:
                if nd == dist[nxt]:
                    preds.setdefault(nxt, []).append((cur, eid))
            else:
                dist[nxt] = nd
                preds.setdefault(nxt, []).append((cur, eid))
                if nxt == dst:
                    sd = nd
                if nd < max_hops:
                    queue.append(nxt)
    if dst not in preds:
        return []
    out, stack = [], [(dst, [], [dst])]
    while stack:
        node, edges, nodes = stack.pop()
        if node == src and edges:
            out.append((edges, nodes) if is_cycle else (edges[::-1], nodes[::-1]))
            continue
        for prev, eid in preds.get(node, []):
            stack.append((prev, edges + [eid], nodes + [prev]))
    return out


class LevelSync:
    """the statement all_shortest_paths.cu runs, for one pair: forward levels with ranks (a level cut into pieces of at most
    `budget` candidates, each piece marking its vertices before the next), the backward predecessor lists, saturating counts and
    suffix sums, and path r unranked from dst"""

    def __init__(self, g, both, max_hops, src, dst, budget=None):
        self.src, self.dst, self.sd = src, dst, 0
        max_hops = (1 << 64) if max_hops is None else max_hops
        front, seen, levels = [src], {src}, []
        L = 0
        while L < max_hops and front:
            levels.append({v: r for r, v in enumerate(front)})
            found, nxt, i0 = False, [], 0
            while i0 < len(front):                          # pieces of consecutive front entries
                i1, size = i0 + 1, len(g.adj(front[i0], both))
                while budget is not None and i1 < len(front) and size + len(g.adj(front[i1], both)) <= budget:
                    size += len(g.adj(front[i1], both))
                    i1 += 1
                if budget is None:
                    i1 = len(front)
                cands = [(e[1] if e[0] == u else e[0]) for u in front[i0:i1] for e in g.adj(u, both)]
                found |= dst in cands
                new = {}
                for v in cands:                             # (rank, position) order: the first to reach v leads
                    if v not in seen and v not in new:
                        new[v] = True
                seen |= set(new)
                nxt += list(new)
                i0 = i1
            L += 1
            if found:
                self.sd = L
                break
            front = nxt
        self.preds, self.cnt, self.suf = {}, {}, {}
        if not self.sd:
            return
        anc = {self.sd: [dst]}
        for l in range(self.sd, 0, -1):
            below = levels[l - 1]
            nxt = set()
            for v in anc[l]:
                ents = [(below[u], t, h, q, u, eid) for q, (u, eid, t, h) in enumerate(g.rev(v, both)) if u in below]
                ents.sort(key=lambda x: x[:3])              # stable: (rank(u), type, half), then fetch order
                self.preds[(l, v)] = [(x[4], x[5]) for x in ents]
                nxt |= {x[4] for x in ents}
            anc[l - 1] = sorted(nxt)
        self.cnt[(0, src)] = 1
        for l in range(1, self.sd + 1):
            for v in anc[l]:
                c, s = 0, []
                for u, _ in reversed(self.preds[(l, v)]):
                    c = min(SAT, c + self.cnt[(l - 1, u)])
                    s.append(c)
                self.suf[(l, v)] = s[::-1]
                self.cnt[(l, v)] = c

    def count(self):
        return self.cnt.get((self.sd, self.dst), 0) if self.sd else 0

    def path(self, r):
        L, v, cyc = self.sd, self.dst, self.src == self.dst
        edges, nodes = [], [v]
        for l in range(L, 0, -1):
            suf, pl = self.suf[(l, v)], self.preds[(l, v)]
            j = max(k for k in range(len(suf)) if r < suf[k])
            if j + 1 < len(suf):
                r -= suf[j + 1]
            u, eid = pl[j]
            edges.append(eid)
            nodes.append(u)
            v = u
        return (edges, nodes) if cyc else (edges[::-1], nodes[::-1])


def windows(counts, lens, first, cap):
    """B200_all_shortest_paths' fill rule: pairs in order from first[i]; stop at the first path that no longer fits"""
    w, e, stop = [], 0, False
    for c, ln, f in zip(counts, lens, first):
        avail, k = max(0, c - f), 0
        if not stop and avail:
            k = min(avail, (cap - e) // ln)
            stop = k < avail
        w.append(k)
        e += k * ln
    return w


def random_graph(rng, n, ntypes):
    rels, eid = {}, 0
    for t in range(ntypes):
        r = []
        for _ in range(int(rng.integers(0, 3 * n))):
            u, v = int(rng.integers(0, n)), int(rng.integers(0, n))
            for _ in range(1 + (rng.random() < 0.15)):     # parallel edges of one type
                r.append((u, v, eid))
                eid += 1
        if rng.random() < 0.5:                               # self-loops
            u = int(rng.integers(0, n))
            r.append((u, u, eid))
            eid += 1
        rels[f"T{t}"] = r
    return rels


def test_transcription_against_the_flow_goldens():
    gold = json.load(open(GOLDEN))
    for case in gold["cases"]:
        gr = gold["graphs"][case["graph"]]
        g = Graph({t: [tuple(e) for e in r] for t, r in gr["types"].items()}, list(gr["types"]))
        paths = expand_row(g, not case["directed"], None, case["src"], case["dst"])
        nodes = [p[1][::-1] if case["reversed"] else p[1] for p in paths]
        assert sorted(nodes) == case["sorted_nodes"], case["name"]
        if "edges_in_order" in case:
            assert [p[0] for p in paths] == case["edges_in_order"], case["name"]
        if "nodes_in_order" in case:
            assert nodes == case["nodes_in_order"], case["name"]
        ls = LevelSync(g, not case["directed"], None, case["src"], case["dst"])
        assert [ls.path(r) for r in range(ls.count())] == paths, case["name"]


def test_level_synchronous_statement_equals_the_transcription():
    rng = np.random.default_rng(2026)
    total = 0
    for k in range(1200):
        n = int(rng.integers(3, 12))
        ntypes = int(rng.integers(1, 4))
        rels = random_graph(rng, n, ntypes)
        order = [f"T{t}" for t in rng.permutation(ntypes)]
        if rng.random() < 0.3:
            order.append("missing")                          # a named type the graph lacks: dropped
        g = Graph(rels, order)
        both = bool(k % 2)
        max_hops = [1, 2, 3, INF][(k // 2) % 4]
        pairs = [(int(rng.integers(0, n)), int(rng.integers(0, n))) for _ in range(5)] + [(0, 0)]
        want_all, lens, counts = [], [], []
        for s, d in pairs:
            want = expand_row(g, both, max_hops, s, d)
            assert len({len(p[0]) for p in want}) <= 1                # every path of a pair has the same length
            budget = [None, 1, 2, 5][k % 4]
            ls = LevelSync(g, both, max_hops, s, d, budget)
            assert ls.count() == len(want)
            assert [ls.path(r) for r in range(ls.count())] == want, (k, s, d, both, max_hops, budget)
            want_all.append(want)
            lens.append(len(want[0][0]) if want else 0)
            counts.append(len(want))
            total += len(want)
        # draining in windows of every size reproduces the single-call lists, across pair boundaries
        for cap in range(1, 1 + max(1, sum(c * ln for c, ln in zip(counts, lens)))):
            if cap < max(lens):
                continue
            first, got = [0] * len(pairs), [[] for _ in pairs]
            while any(f < c for f, c in zip(first, counts)):
                w = windows(counts, lens, first, cap)
                assert sum(w) > 0
                for i, ki in enumerate(w):
                    got[i] += want_all[i][first[i]:first[i] + ki]
                    first[i] += ki
            assert got == want_all
    assert total > 3000


def test_unranking_at_saturated_counts():
    """a chain of 70 diamonds has 2^70 shortest paths: the count saturates, and paths unranked at ranks near 2^64 - 2 are valid,
    distinct and of the right length"""
    k = 70
    rels, eid, hub = [], 0, 0
    for i in range(k):
        a, b, nh = hub + 1, hub + 2, hub + 3
        for u, v in ((hub, a), (hub, b), (a, nh), (b, nh)):
            rels.append((u, v, eid))
            eid += 1
        hub = nh
    g = Graph({"R": rels}, ["R"])
    ends = {e[2]: (e[0], e[1]) for e in rels}
    for both in (False, True):
        ls = LevelSync(g, both, None, 0, hub)
        assert ls.count() == SAT
        seen = set()
        for r in [SAT - 2, SAT - 3, SAT - 100, (1 << 63) + 5, 0, 1]:
            edges, nodes = ls.path(r)
            assert len(edges) == 2 * k and nodes[0] == 0 and nodes[-1] == hub
            for e, u, v in zip(edges, nodes, nodes[1:]):
                assert set(ends[e]) == {u, v}
            seen.add(tuple(edges))
        assert len(seen) == 6
    small = Graph({"R": rels[:4 * 10]}, ["R"])
    ls = LevelSync(small, False, None, 0, 30)
    assert [ls.path(r) for r in range(ls.count())] == expand_row(small, False, None, 0, 30) and ls.count() == 1 << 10


def test_self_loop_on_src_is_a_one_edge_cycle():
    g = Graph({"R": [(0, 0, 5), (0, 1, 6), (1, 0, 7), (0, 0, 9)], "S": [(0, 0, 8)]}, ["R", "S"])
    for both in (False, True):
        want = expand_row(g, both, None, 0, 0)
        assert [p[0] for p in want] == [[8], [9], [5]] and all(p[1] == [0, 0] for p in want)
        ls = LevelSync(g, both, None, 0, 0)
        assert [ls.path(r) for r in range(ls.count())] == want


def call(src, dst, types, dir=fb.DIR_OUT, max_hops=SAT, ntypes=None, cap=64, out=True, edges=True, first=None):
    s, d = np.asarray(src, np.uint64), np.asarray(dst, np.uint64)
    n = len(s)
    count, ln, p = np.zeros(max(1, n), np.uint64), np.zeros(max(1, n), np.uint32), np.zeros(n + 1, np.uint64)
    pe, pn = np.zeros(max(cap, 1), np.uint64), np.zeros(2 * max(cap, 1), np.uint32)
    ne = U64(0)
    f = None if first is None else np.asarray(first, np.uint64)
    info = lib().B200_all_shortest_paths(s.ctypes.data if n else None, d.ctypes.data if n else None, n, _layers(types),
                                         len(types) if ntypes is None else ntypes, dir, max_hops, None if f is None else f.ctypes.data,
                                         count.ctypes.data, ln.ctypes.data, p.ctypes.data if out else None,
                                         pe.ctypes.data if edges else None, pn.ctypes.data, cap, C.byref(ne))
    return info, count[:n], ln[:n], p, ne.value


def tensor(n=16, huge=False):
    nn = 1 << 60 if huge else n
    return {"m": Matrix(nn, nn, "u64"), "dp": Matrix(nn, nn, "u64"), "dm": Matrix(nn, nn), "mt": Matrix(nn, nn),
            "mt_dp": Matrix(nn, nn), "mt_dm": Matrix(nn, nn)}


def test_argument_errors():
    fb.init()
    t, small = tensor(), tensor(8)
    assert call([0], [1], [t], out=False)[0] == -2                          # GrB_NULL_POINTER: out_p
    assert call([0], [1], [dict(t, m=None)])[0] == -2                       # m
    assert call([0], [1], [dict(t, mt=None)])[0] == -2                      # mt, needed in both directions
    assert call([0], [1], [dict(t, mt=None)], dir=fb.DIR_BOTH)[0] == -2
    for nt in (0, 65537):
        assert call([0], [1], [t], ntypes=nt)[0] == -3                      # GrB_INVALID_VALUE: ntypes
    for d in (fb.DIR_IN, 3, -1):
        assert call([0], [1], [t], dir=d)[0] == -3                          # dir not OUT / BOTH
    assert call([0], [1], [dict(t, m=Matrix(16, 16))])[0] == -5             # GrB_DOMAIN_MISMATCH: m not UINT64
    assert call([0], [1], [dict(t, dp=Matrix(16, 16))])[0] == -5            # dp not UINT64
    assert call([0], [1], [t, small])[0] == -6                              # GrB_DIMENSION_MISMATCH
    assert call([0], [1], [dict(t, mt=Matrix(16, 8))])[0] == -6
    assert call([16], [1], [t])[0] == -4                                    # GrB_INVALID_INDEX
    assert call([0], [16], [t])[0] == -4
    assert call([0], [1], [tensor(huge=True)])[0] == -8                     # GrB_NOT_IMPLEMENTED: host-resident layers


def test_empty_calls_do_no_device_work():
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    t["mt"].set(1, 0, True)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    info, count, ln, p, ne = call([], [], [t])
    assert info == 0 and p.tolist() == [0] and ne == 0
    info, count, ln, p, ne = call([0, 1], [1, 1], [t], max_hops=0, first=[3, 4])
    assert info == 0 and count.tolist() == [0, 0] and ln.tolist() == [0, 0] and p.tolist() == [0, 0, 0] and ne == 0
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before


@pytest.mark.skipif(_has_gpu(), reason="only meaningful on a box without a GPU")
def test_all_shortest_paths_fails_loudly_without_gpu():
    fb.init()
    t = tensor()
    t["m"].set(0, 1, 7)
    before = fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")
    for d in (fb.DIR_OUT, fb.DIR_BOTH):
        for hi in (1, SAT):
            assert call([0, 1, 2], [1, 1, 3], [t], dir=d, max_hops=hi)[0] == -7002   # GxB_GPU_ERROR
            assert call([0, 1, 2], [1, 1, 3], [t], dir=d, max_hops=hi, edges=False)[0] == -7002
    assert (fb.get_stat("h2d_bytes"), fb.get_stat("d2h_bytes"), fb.get_stat("launches")) == before
    assert t["m"].pending()                                                  # the queued write was not finished by the call
    with pytest.raises(fb.GrbError) as e:
        fb.all_shortest_paths([0], [1], [t])
    assert e.value.info == -7002
