"""Golden fixture of the random walk kernels: K from the real reference (oracle/_ref, GraKeL 0.1.11 with its lamda
tuning) on every row of the route table -> tests/golden/random_walk.npz.

Each case stores its graphs as the reference's dense adjacency matrices (inputs are rebuilt as [A, {index: label}]),
the labels, the parameters (JSON), K of fit_transform and, for transform cases, K of transform, plus the warnings the
reference raised.  `dict_inputs` pins the vertex set and matrix of edge-dictionary spellings against
Graph(g, {}, {}, "adjacency").get_adjacency_matrix().

    python tests/golden/make_golden_random_walk.py
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
sys.path.insert(0, HERE)


def mutag(n):
    import gio
    X = gio.dec_dataset(gio.load(os.path.join(HERE, "mutag_graphs.json.gz")))[:n]
    from grakel.graph import Graph
    out = []
    for x in X:
        g = Graph(x[0], x[1], {}, "adjacency")
        A = g.get_adjacency_matrix()
        L = g.get_labels(purpose="adjacency")
        out.append((np.asarray(A, dtype=float), [L[i] for i in range(A.shape[0])]))
    return out


def synthetic(seed, n_graphs, signed=False, directed=False, loops=False, scale=1.0):
    rs = np.random.RandomState(seed)
    out = []
    for g in range(n_graphs):
        n = [1, 2, 3, 5, 7, 9][g % 6] if g < 6 else int(rs.randint(2, 10))
        A = (rs.rand(n, n) < 0.35).astype(float)
        if not directed:
            A = np.triu(A, 1)
            A = A + A.T
        elif not loops:
            np.fill_diagonal(A, 0)
        if loops:
            A[np.diag_indices(n)] = rs.rand(n) < 0.3
        if signed:
            W = rs.choice([0.5, 1.0, 2.0, -1.0, -0.25], size=(n, n))
            if not directed:
                W = np.triu(W) + np.triu(W, 1).T
            A = A * W
        A = A * scale
        if n >= 4:  # an isolated vertex
            A[n - 1, :] = 0
            A[:, n - 1] = 0
        out.append((A, [int(rs.randint(3)) for _ in range(n)]))
    return out


def cases():
    m = mutag(24)
    sym = synthetic(1, 10)
    dirw = synthetic(2, 10, signed=True, directed=True, loops=True)
    symw = synthetic(3, 10, signed=True)
    nonneg = synthetic(4, 10, directed=True, loops=True)
    big = synthetic(5, 4, scale=3.0)
    disjoint = [(np.array([[0., 1.], [1., 0.]]), [0, 0]), (np.array([[0., 1.], [1., 0.]]), [1, 1]),
                (np.array([[0., 1., 0.], [1., 0., 1.], [0., 1., 0.]]), [0, 1, 0])]
    C = []
    add = lambda name, cls, params, X, Y=None: C.append((name, cls, params, X, Y))
    add("mutag_rw_test_lamda", "RW", dict(lamda=0.01), m)
    add("mutag_rwl_test_lamda", "RWL", dict(lamda=1e-4, normalize=True), m)
    add("mutag_rw_default", "RW", dict(normalize=True), m)
    add("mutag_rwl_default", "RWL", dict(), m)
    add("directed_signed_cg", "RW", dict(lamda=0.02), dirw[:7], dirw[7:])
    add("directed_signed_cg_labeled", "RWL", dict(lamda=0.02, normalize=True), dirw[:7], dirw[7:])
    add("diverging_lamda", "RW", dict(lamda=0.5), sym)
    add("transform_larger_radius", "RW", dict(lamda=0.05), sym[:6], big)
    add("empty_label_intersection", "RWL", dict(lamda=0.1), disjoint)
    add("fast_p_geometric", "RW", dict(lamda=0.1, p=3), symw[:7], symw[7:])
    add("fast_p_exponential", "RW", dict(lamda=0.3, p=4, kernel_type="exponential", normalize=True), dirw)
    add("fast_exponential", "RW", dict(lamda=0.2, kernel_type="exponential"), symw[:7], symw[7:])
    add("fast_exponential_directed", "RW", dict(lamda=0.2, kernel_type="exponential", normalize=True), dirw)
    add("baseline_p", "RW", dict(lamda=0.1, p=3, method_type="baseline", normalize=True), dirw[:7], dirw[7:])
    add("baseline_exponential", "RW", dict(lamda=0.1, kernel_type="exponential", method_type="baseline"), nonneg)
    add("baseline_geometric_symmetric", "RW", dict(lamda=0.02, method_type="baseline", normalize=True), symw[:7], symw[7:])
    add("baseline_p_labeled", "RWL", dict(lamda=0.1, p=2, method_type="baseline"), dirw[:7], dirw[7:])
    add("fast_p_labeled", "RWL", dict(lamda=0.1, p=3, normalize=True), symw)
    add("fast_exponential_labeled", "RWL", dict(lamda=0.3, kernel_type="exponential"), nonneg[:7], nonneg[7:])
    add("baseline_exponential_labeled", "RWL", dict(lamda=0.2, kernel_type="exponential", method_type="baseline",
                                                     normalize=True), nonneg)
    return C


def dict_inputs():
    return [
        {0: [1], 1: [0, 2], 2: [], 7: []},
        {(0, 1): 2.0, (1, 0): -1.5, (2, 2): 0.5, (4, 0): 0.0},
        {"a": {"b": 1.0, "c": -2.0}, "c": {}, "d": {}},
        [(3, 1), (1, 3), (5, 5)],
        [(0, 2, 0.5), (2, 0, 0.5), (0, 2, 4.0)],
    ]


def as_input(G):
    return [[A, dict(enumerate(L))] for A, L in G]


def flat(G):
    sizes = np.array([A.shape[0] for A, _ in G], dtype=np.int64)
    A = np.concatenate([A.ravel() for A, _ in G]) if G else np.zeros(0)
    L = np.array([l for _, L in G for l in L], dtype=np.int64)
    return sizes, A, L


def unflat(sizes, A, L):
    out, a, v = [], 0, 0
    for n in sizes.tolist():
        out.append((A[a:a + n * n].reshape(n, n), L[v:v + n].tolist()))
        a += n * n
        v += n
    return out


def main():
    from grakel.graph import Graph
    from grakel.kernels import RandomWalk, RandomWalkLabeled
    out = {}
    for name, cls, params, X, Y in cases():
        est = (RandomWalk if cls == "RW" else RandomWalkLabeled)(**params)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            K = est.fit_transform(as_input(X))
            Kt = est.transform(as_input(Y)) if Y is not None else None
        msgs = [str(x.message) for x in w if issubclass(x.category, RuntimeWarning)]
        meta = dict(cls=cls, params=params, warnings=msgs, lamda_used=est._lamda)
        out[name + "/meta"] = np.array(json.dumps(meta))
        for k, v in zip(("sizes", "A", "L"), flat(X)):
            out[name + "/X_" + k] = v
        out[name + "/K"] = K
        if Y is not None:
            for k, v in zip(("sizes", "A", "L"), flat(Y)):
                out[name + "/Y_" + k] = v
            out[name + "/Kt"] = Kt
        print(name, K.shape, "transform" if Y is not None else "", msgs and "warned")
    for i, g in enumerate(dict_inputs()):
        out["dict/%d" % i] = Graph(g, {}, {}, "adjacency").get_adjacency_matrix()
    np.savez_compressed(os.path.join(HERE, "random_walk.npz"), **out)


if __name__ == "__main__":
    main()
