"""CPU restatement of the reference's GraphletSampling, sampled route (graphlet_sampling.py), written from its
description: the draws on a numpy RandomState, the class of each sample as the least bit pattern over the relabelings
of its undirected graph (loops included), the bins' counts with the first graph's exception, and K in float64."""
from itertools import permutations

import numpy as np


def n_samples_of(sampling, k):
    if "n_samples" in sampling:
        return sampling["n_samples"]
    delta, epsilon, a = sampling.get("delta", 0.05), sampling.get("epsilon", 0.05), sampling.get("a", -1)
    if a == -1:
        a = {3: 4, 4: 8, 5: 19, 6: 53}[k]
    return int(np.ceil(2 * (a * np.log10(2) + np.log10(1 / delta)) / (epsilon ** 2)))


def draws(A, k, n_samples, rs):
    """The vertex index arrays of one graph's samples."""
    n = A.shape[0]
    lo, hi = min(3, n), min(k, n)
    out = []
    for _ in range(n_samples):
        r = lo if lo == hi else rs.randint(lo, hi + 1)
        out.append(rs.choice(list(range(n)), r, replace=False))
    return out


def pattern(Q):
    """Bits of the undirected graph of Q: pairs i < j in row-major order, then the loops."""
    m = Q.shape[0]
    bits, b = 0, 0
    for i in range(m):
        for j in range(i + 1, m):
            if Q[i, j] or Q[j, i]:
                bits |= 1 << b
            b += 1
    for i in range(m):
        if Q[i, i]:
            bits |= 1 << (b + i)
    return bits


_CANON = {}


def class_code(Q):
    """(size, least pattern over the relabelings): one value per isomorphism class."""
    m = Q.shape[0]
    key = (m, pattern(Q))
    if key not in _CANON:
        _CANON[key] = (m, min(pattern(Q[np.ix_(p, p)]) for p in permutations(range(m))))
    return _CANON[key]


def canon_patterns(m, pats):
    """Least pattern over the m! relabelings of each pattern of `pats` (same bit layout as `pattern`), vectorised."""
    pairs = [(i, j) for i in range(m) for j in range(i + 1, m)]
    P = len(pairs)
    at = {pq: b for b, pq in enumerate(pairs)}
    pats = np.asarray(pats, dtype=np.int64)
    best = pats.copy()
    for perm in permutations(range(m)):
        dst = [at[tuple(sorted((perm[i], perm[j])))] for i, j in pairs] + [P + perm[i] for i in range(m)]
        out = np.zeros_like(pats)
        for b, d in enumerate(dst):
            out |= ((pats >> b) & 1) << d
        best = np.minimum(best, out)
    return best


def classes_of_draws(A, size, idx):
    """The class of every sample of one graph from its drawn sizes and concatenated indexes, vectorised over the
    samples of one size (for large sample counts)."""
    off = np.concatenate([[0], np.cumsum(size, dtype=np.int64)]).astype(np.int64)
    out = [None] * len(size)
    A = np.asarray(A) > 0
    for m in (int(x) for x in np.unique(size)):
        at = np.nonzero(size == m)[0]
        ix = off[at][:, None] + np.arange(m)[None, :]
        V = np.asarray(idx)[ix] if m else np.zeros((len(at), 0), dtype=np.int64)
        bits = np.zeros(len(at), dtype=np.int64)
        b = 0
        for i in range(m):
            for j in range(i + 1, m):
                bits |= (A[V[:, i], V[:, j]] | A[V[:, j], V[:, i]]).astype(np.int64) << b
                b += 1
        for i in range(m):
            bits |= A[V[:, i], V[:, i]].astype(np.int64) << (b + i)
        uniq, inv = np.unique(bits, return_inverse=True)
        canon = [(m, int(c)) for c in canon_patterns(m, uniq)]
        for t, u in zip(at.tolist(), inv.tolist()):
            out[t] = canon[u]
    return out


def graph_classes(A, k, n_samples, rs):
    return [class_code(A[np.ix_(ix, ix)]) for ix in draws(A, k, n_samples, rs)]


def counts(classes_per_graph, fitted=()):
    """[{class: count}] with the reference's rule: samples, + 1 unless the graph is the first (in order) with the
    class; a class in `fitted` (the fit's classes, in a transform) always gets the + 1."""
    first = {}
    out = []
    for g, cl in enumerate(classes_per_graph):
        c = {}
        for x in cl:
            c[x] = c.get(x, 0) + 1
        for x in c:
            if x in fitted:
                c[x] += 1
            elif first.setdefault(x, g) != g:
                c[x] += 1
        out.append(c)
    return out


def gram(rows, cols):
    classes = sorted(set().union(*cols) if cols else set())
    at = {x: i for i, x in enumerate(classes)}
    X = np.zeros((len(cols), len(classes)))
    for i, c in enumerate(cols):
        for x, v in c.items():
            X[i, at[x]] = v
    Y = np.zeros((len(rows), len(classes)))
    for i, c in enumerate(rows):
        for x, v in c.items():
            if x in at:
                Y[i, at[x]] = v
    return Y @ X.T


def diag(rows):
    return np.array([float(sum(v * v for v in c.values())) for c in rows])


def fit_transform(X, k, sampling, rs, normalize=False):
    n = n_samples_of(sampling, k)
    cx = counts([graph_classes(A, k, n, rs) for A in X])
    K = gram(cx, cx)
    if normalize:
        d = diag(cx)
        with np.errstate(divide="ignore", invalid="ignore"):
            K = K / np.sqrt(np.outer(d, d))
    return K, cx


def transform(Y, cx, k, sampling, rs, normalize=False):
    n = n_samples_of(sampling, k)
    fitted = set().union(*cx)
    cy = counts([graph_classes(A, k, n, rs) for A in Y], fitted)
    K = gram(cy, cx)
    if normalize:
        with np.errstate(divide="ignore", invalid="ignore"):
            K = K / np.sqrt(np.outer(diag(cy), diag(cx)))
    return K, cy
