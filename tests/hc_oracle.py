"""NumPy restatement of HadamardCode over VertexHistogram (grakel/kernels/hadamard_code.py): int64 vectors whose
additions wrap, classes by np.unique over the rows, per-level histograms, K = sum of the level Grams."""
import numpy as np


def hadamard_row(r, W):
    """Row r of Sylvester's W x W Hadamard matrix: (-1)^popcount(r & c)."""
    c = np.arange(W, dtype=np.int64) & int(r)
    odd = np.zeros(W, dtype=np.int64)
    while c.any():
        odd ^= c & 1
        c >>= 1
    return np.where(odd == 1, -1, 1).astype(np.int64)


def edge_dictionary(g):
    """{key: [out-neighbours]} of the reference's edge dictionary (graph.py:1182-1204)."""
    if isinstance(g, np.ndarray) or (type(g) is list and all(isinstance(r, list) for r in g)):
        A = np.asarray(g)
        return {i: np.flatnonzero(A[i] > 0).tolist() for i in range(A.shape[0])}
    out = {}
    if type(g) is dict and all(type(k) is tuple for k in g):
        items = list(g)
    elif type(g) is dict and all(isinstance(d, list) for d in g.values()):
        items = [(u, v) for u, lst in g.items() for v in lst]
    elif type(g) is dict:
        for u in g:
            out.setdefault(u, [])
        items = [(u, v) for u, d in g.items() for v in d]
    else:
        items = [(t[0], t[1]) for t in g]
    for u, v in items:
        out.setdefault(u, [])
        out.setdefault(v, [])
        if v not in out[u]:
            out[u].append(v)
    return out


def enumerate_labels(label_dicts, enum=None):
    enum = {} if enum is None else dict(enum)
    for L in label_dicts:
        for v in set(L.values()):
            if v not in enum:
                enum[v] = len(enum)
    return enum


def levels(X, n_iter, enum):
    """Per level, one {vertex: int64 vector} per graph."""
    nl = len(enum)
    W = 1 if nl <= 1 else 1 << (nl - 1).bit_length()
    rows = {r: hadamard_row(r, W) for r in set(enum.values())}
    cur = [{k: rows[enum[v]] for k, v in x[1].items()} for x in X]
    out = [cur]
    nbrs = [edge_dictionary(x[0]) for x in X]
    for _ in range(1, n_iter):
        nxt = []
        for old, nb in zip(cur, nbrs):
            d = {}
            for k, ns in nb.items():
                s = old[k].copy()
                for q in ns:
                    s = s + old[q]  # int64 array addition wraps
                d[k] = s
            nxt.append(d)
        cur = nxt
        out.append(cur)
    return out


def packed_rows(X, level, W):
    """[V, W] rows of one level in packed order (labels dictionary key order), zeros where absent."""
    rows = []
    for x, d in zip(X, level):
        for k in x[1]:
            rows.append(d[k] if k in d else np.zeros(W, dtype=np.int64))
    return np.array(rows, dtype=np.int64).reshape(-1, W)


def kernel(X, n_iter, Y=None):
    """(K of fit_transform, or of transform against X when Y is given, fitted enumeration).  Same-width Y only."""
    enum = enumerate_labels(x[1] for x in X)
    full = list(X) + (list(Y) if Y is not None else [])
    if Y is not None:
        enum_all = enumerate_labels((y[1] for y in Y), enum)
    else:
        enum_all = enum
    lv = levels(full, n_iter, enum_all)
    nx, n = len(X), len(full)
    K = np.zeros((n, n))
    for level in lv:
        vecs = [np.array(list(d.values()), dtype=np.int64).reshape(len(d), -1) for d in level]
        allv = np.concatenate(vecs)
        if not len(allv):
            continue
        _, inv = np.unique(allv, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        gid = np.repeat(np.arange(n), [len(v) for v in vecs])
        H = np.zeros((n, inv.max() + 1))
        np.add.at(H, (gid, inv), 1.0)
        K += H @ H.T
    if Y is None:
        return K, enum
    return K[nx:, :nx], enum
