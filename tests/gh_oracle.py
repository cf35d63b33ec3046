"""NumPy restatement of GraphHopper (grakel/kernels/graph_hopper.py) for the tests.

The node maps follow the DAG rule of DESIGN §4.9 with breadth-first distances: for a root j, u -> v is a DAG edge
when D_j(u) = D_j(v) - 1 and either v -> u is an edge (an out-neighbour of v one level up) or u is the smallest-id
in-neighbour of v one level up and u is not the smallest vertex id j reaches.  sigma_j(v) counts DAG paths from j,
des_j(v, l) DAG paths of length l leaving v, and M[v, a, b] = sum_j [a = D_j(v)] sigma_j(v) des_j(v, b - a).
Vertices that reach nothing but themselves contribute M[v, 0, 0] += 1 (the reference raises there)."""
from collections import deque

import numpy as np


def adjacency_of(x):
    """Dense adjacency (entries > 0 are edges) and n x d attributes of a reference-style (adjacency, labels) element."""
    A = np.asarray(x[0], dtype=float)
    L = x[1]
    attrs = np.array([np.asarray(L[i], dtype=float).ravel() for i in range(A.shape[0])])
    return A, attrs


def diameter(A):
    n = A.shape[0]
    best = 0
    for j in range(n):
        D = bfs(A, j)
        best = max(best, int(D[D >= 0].max()))
    return best


def bfs(A, j):
    n = A.shape[0]
    D = -np.ones(n, dtype=np.int64)
    D[j] = 0
    q = deque([j])
    while q:
        u = q.popleft()
        for w in np.nonzero(A[u] > 0)[0]:
            if w != u and D[w] < 0:
                D[w] = D[u] + 1
                q.append(w)
    return D


def node_maps(A, delta):
    """n x delta x delta maps M of one graph."""
    n = A.shape[0]
    E = (A > 0) & ~np.eye(n, dtype=bool)
    M = np.zeros((n, delta, delta))
    for j in range(n):
        D = bfs(A, j)
        reach = np.nonzero(D >= 0)[0]
        minr = int(reach.min())
        ecc = int(D.max())
        parents = {}
        for v in reach:
            if v == j:
                continue
            up = [u for u in reach if D[u] == D[v] - 1]
            P = {u for u in up if E[v, u]}
            ins = [u for u in up if E[u, v]]
            if ins and min(ins) != minr:
                P.add(min(ins))
            parents[v] = P
        sigma = np.zeros(n, dtype=np.int64)
        sigma[j] = 1
        for v in sorted(reach, key=lambda v: D[v]):
            if v != j:
                sigma[v] = sum(sigma[u] for u in parents[v])
        des = np.zeros((n, ecc + 1), dtype=np.int64)
        des[reach, 0] = 1
        for v in sorted(reach, key=lambda v: -D[v]):
            if v == j:
                continue
            for u in parents[v]:
                des[u, 1:] += des[v, :-1]
        for v in reach:
            a = int(D[v])
            for l in range(ecc - a + 1):
                M[v, a, a + l] += float(sigma[v] * des[v, l])
    return M


def gaussian(mu):
    return lambda xi, xj: np.exp(-mu * np.sum((xi[:, None, :] - xj[None, :, :]) ** 2, axis=2))


def bridge(xi, xj):
    return np.maximum(0.0, (4.0 - np.sqrt(np.sum((xi[:, None, :] - xj[None, :, :]) ** 2, axis=2))) / 4.0)


def linear(xi, xj):
    return xi @ xj.T


def node_kernel(kernel_type):
    if kernel_type == "linear":
        return linear
    if kernel_type == "gaussian":
        return gaussian(1.0)
    if kernel_type == "bridge":
        return bridge
    if isinstance(kernel_type, tuple) and kernel_type[0] == "gaussian":
        return gaussian(float(kernel_type[1]))
    raise ValueError(kernel_type)


class GraphHopperOracle:
    """fit_transform / transform of GraphHopper over reference-style (adjacency, attribute dict) elements."""

    def __init__(self, kernel_type="linear", normalize=False):
        self.k = node_kernel(kernel_type)
        self.normalize = normalize

    def _maps(self, X, delta=None):
        G = [adjacency_of(x) for x in X]
        d = max(diameter(A) for A, _ in G) + 1
        delta = d if delta is None else max(delta, d)
        return [(node_maps(A, delta).reshape(A.shape[0], -1), at) for A, at in G], d, delta

    def _pair(self, x, y):
        return float(np.sum((x[0] @ y[0].T) * self.k(x[1], y[1])))

    def fit_transform(self, X):
        self.X_, self.delta_, _ = self._maps(X)
        n = len(self.X_)
        K = np.zeros((n, n))
        for i in range(n):
            for j in range(i, n):
                K[i, j] = K[j, i] = self._pair(self.X_[i], self.X_[j])
        self.xdiag_ = np.diagonal(K).copy()
        if self.normalize:
            with np.errstate(invalid="ignore", divide="ignore"):
                K = K / np.sqrt(np.outer(self.xdiag_, self.xdiag_))
        return K

    def transform(self, Y):
        Ym, _, width = self._maps(Y, self.delta_)
        w = self.delta_
        X = [(m.reshape(-1, w, w), a) for m, a in self.X_]
        pad = []
        for m, a in X:  # X's maps are zero beyond its delta: pad to Y's width
            mm = np.zeros((m.shape[0], width, width))
            mm[:, :w, :w] = m
            pad.append((mm.reshape(m.shape[0], -1), a))
        K = np.array([[self._pair(y, x) for x in pad] for y in Ym]).reshape(len(Ym), len(pad))
        self.ydiag_ = np.array([self._pair(y, y) for y in Ym])
        if self.normalize:
            with np.errstate(invalid="ignore", divide="ignore"):
                K = K / np.sqrt(np.outer(self.ydiag_, self.xdiag_))
        return K
