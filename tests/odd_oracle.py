"""CPU restatement of OddSth (the reference's odd_sth.py) in priority-queue form, for the host and device tests.

Each graph is packed as the estimator packs it (grakel_b200.packing.pack, mode "sp", neighbours in edge-dictionary
order); every vertex roots a DAG: the BFS over the out-neighbours cut at depth h, an edge u -> w when w is one level
below u.  Kahn's algorithm pops the least (label rank, insertion sequence) from a heap; a node's identity is
str(label), followed for an inner node by "(" + its children's identities, last popped first, joined by "," + ")"."""
import heapq
from collections import Counter

import numpy as np

from grakel_b200.kernels import odd_label_tables
from grakel_b200.packing import pack


def graph_features(n, rows, strs, ranks, h):
    """Counter of identity strings over every (root, node) pair of one graph (local vertex ids)."""
    out = Counter()
    for root in range(n):
        depth = {root: 0}
        order = [root]
        k = 0
        while k < len(order):
            u = order[k]
            k += 1
            if h is not None and depth[u] >= h:
                continue
            for w in rows[u]:
                if w not in depth:
                    depth[w] = depth[u] + 1
                    order.append(w)
        expanded = {u for u in order if h is None or depth[u] < h}
        children = {u: [w for w in rows[u] if depth.get(w) == depth[u] + 1] if u in expanded else [] for u in order}
        indeg = Counter(w for u in order for w in children[u])
        heap = [(ranks[root], 0, root)]
        seq = 1
        pos = {}
        while heap:
            _, _, u = heapq.heappop(heap)
            pos[u] = len(pos)
            for w in children[u]:
                indeg[w] -= 1
                if indeg[w] == 0:
                    heapq.heappush(heap, (ranks[w], seq, w))
                    seq += 1
        ident = {}
        for u in sorted(order, key=lambda x: -pos[x]):
            ch = sorted(children[u], key=lambda x: -pos[x])
            ident[u] = strs[u] + ("(" + ",".join(ident[w] for w in ch) + ")" if ch else "")
            out[ident[u]] += 1
    return out


def features(X, h=None):
    """phi of every graph of the element list X: a list of Counters."""
    b = pack(X, "sp", need_labels=True, len_ok=lambda n: n >= 2, keep_edge_order=True)
    ids, rank, strings = odd_label_tables(b.labels, b.graph_ptr)
    gp, rp, ci = b.graph_ptr, b.row_ptr, b.col_idx
    out = []
    for g in range(b.n_graphs):
        a, z = int(gp[g]), int(gp[g + 1])
        rows = [[int(w) - a for w in ci[rp[v]:rp[v + 1]]] for v in range(a, z)]
        strs = [strings[i] for i in ids[a:z]]
        out.append(graph_features(z - a, rows, strs, rank[a:z].tolist(), h))
    return out


def first_counts(phis):
    """C[f]: the count of f in the first graph that has it."""
    C = {}
    for p in phis:
        for f, c in p.items():
            C.setdefault(f, c)
    return C


def kernel(X, Y=None, h=None, normalize=False):
    """fit_transform(X) or, with Y, transform(Y) after fit(X); exact integers in fp64."""
    px = features(X, h)
    return gram(px, None if Y is None else features(Y, h), normalize)


def gram(px, py=None, normalize=False):
    """kernel() of the feature Counters of the fitted graphs (px) and of the transformed ones (py, None for
    fit_transform).  The sums are exact: int64 sparse products when every self similarity, and so (Cauchy-Schwarz)
    every entry, stays below 2^62 (thousands of graphs), Python integers otherwise."""
    C = first_counts(px + ([] if py is None else py))
    py_ = px if py is None else py
    col = {f: i for i, f in enumerate(C)}
    if max([sum(C[f] * c * c for f, c in p.items()) for p in px + py_] or [0]) < 2 ** 62:
        from scipy.sparse import csr_matrix

        def mat(ps):
            rows = [i for i, p in enumerate(ps) for _ in p]
            cols = [col[f] for p in ps for f in p]
            vals = [c for p in ps for c in p.values()]
            return csr_matrix((np.array(vals, dtype=np.int64), (rows, cols)), shape=(len(ps), len(col)))
        cw = np.array(list(C.values()), dtype=np.int64)
        ax, ay = mat(px), mat(py_)
        K = np.asarray((ay.multiply(cw[None, :]).tocsr() @ ax.T).todense(), dtype=np.int64).astype(np.float64)
        dx = np.asarray(ax.multiply(ax).multiply(cw[None, :]).sum(axis=1), dtype=np.int64).ravel().astype(np.float64)
        dy = np.asarray(ay.multiply(ay).multiply(cw[None, :]).sum(axis=1), dtype=np.int64).ravel().astype(np.float64)
    else:
        K = np.array([[sum(C[f] * c * q.get(f, 0) for f, c in a.items()) for q in px] for a in py_], dtype=np.float64)
        dx = np.array([sum(C[f] * c * c for f, c in a.items()) for a in px], dtype=np.float64)
        dy = np.array([sum(C[f] * c * c for f, c in a.items()) for a in py_], dtype=np.float64)
    K = K.reshape(len(py_), len(px))
    if normalize:
        K = K / np.sqrt(np.outer(dy, dx))
    return K
