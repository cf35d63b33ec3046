"""GraphletSampling golden cases (sampled route).  Every input is stored in tests/golden/graphlet_sampling.npz as
adjacency matrices beside the reference's results; `element` turns a matrix back into the input form the case used
(adjacency matrix, edge dictionary or Graph object), so the tests need nothing but that file."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graphlet_sampling.npz")

# (name, constructor parameters) whose `fit` raises in the reference's `initialize`
ERROR_CASES = [("k_float", dict(k=5.0, sampling={"n_samples": 5})), ("k_two", dict(k=2, sampling={"n_samples": 5})),
               ("delta_big", dict(sampling={"delta": 2.0})), ("epsilon_negative", dict(sampling={"epsilon": -0.1})),
               ("a_float", dict(sampling={"a": 2.5})), ("a_zero", dict(sampling={"a": 0})),
               ("a_small", dict(sampling={"a": -2})), ("bad_dict", dict(sampling={"x": 1})),
               ("not_dict", dict(sampling=[1, 2])),
               ("n_samples_with_delta", dict(sampling={"n_samples": 5, "delta": 0.1}))]


def rand_adj(rs, n, p, directed=False, loops=0.0):
    M = (rs.rand(n, n) < p).astype(float)
    A = M if directed else np.triu(M, 1)
    A = A - np.diag(np.diag(A))
    if not directed:
        A = A + A.T
    if loops:
        A = A + np.diag((rs.rand(n) < loops).astype(float))
    return A


def graphs(name, seed):
    """The fit and transform graph lists of a case."""
    rs = np.random.RandomState(seed)
    if name == "small":  # fewer than 3 and fewer than k vertices
        X = [rand_adj(rs, n, 0.6) for n in (1, 2, 3, 4, 2, 6, 5)]
        Y = [rand_adj(rs, n, 0.6) for n in (2, 1, 4, 7)]
    elif name == "directed":
        X = [rand_adj(rs, n, 0.3, directed=True) for n in rs.randint(4, 14, size=10)]
        Y = [rand_adj(rs, n, 0.3, directed=True) for n in rs.randint(4, 14, size=6)]
    elif name == "loops":
        X = [rand_adj(rs, n, 0.3, loops=0.4) for n in rs.randint(3, 12, size=10)]
        Y = [rand_adj(rs, n, 0.5, loops=0.5) for n in rs.randint(3, 12, size=6)]
    elif name == "large":  # ids >= 32, degrees >= 8, more than 128 vertices
        X = [rand_adj(rs, n, p) for n, p in ((40, 0.25), (150, 0.05), (36, 0.3), (200, 0.02))]
        Y = [rand_adj(rs, n, p) for n, p in ((45, 0.2), (130, 0.04))]
    else:  # "new_classes": the transform graphs are dense, the fitted ones sparse
        X = [rand_adj(rs, n, 0.15) for n in rs.randint(6, 12, size=8)]
        Y = [rand_adj(rs, n, 0.9, loops=0.3) for n in rs.randint(6, 12, size=5)]
    return X, Y


# (name, graphs, k, sampling, input form, seed)
CASES = [
    ("small_k3", "small", 3, {"n_samples": 20}, "adjacency", 1),
    ("small_k5", "small", 5, {"n_samples": 30}, "dictionary", 2),
    ("directed_k4", "directed", 4, {"n_samples": 50}, "adjacency", 3),
    ("directed_k6", "directed", 6, {"n_samples": 40}, "graph", 4),
    ("loops_k5", "loops", 5, {"n_samples": 60}, "dictionary", 5),
    ("loops_k6", "loops", 6, {"n_samples": 30}, "adjacency", 6),
    ("large_k5", "large", 5, {"n_samples": 200}, "adjacency", 7),
    ("new_classes_k4", "new_classes", 4, {"n_samples": 40}, "graph", 8),
    ("epsilon_k3", "new_classes", 3, {"epsilon": 0.3}, "adjacency", 9),
    ("delta_a_k5", "directed", 5, {"delta": 0.2, "epsilon": 0.4, "a": 3}, "dictionary", 10),
]


def directed(gname):
    """The device path refuses these (non-symmetric adjacency); the oracle only restates undirected samples."""
    return gname == "directed"


def element(A, form, Graph):
    """A as the case's input form: the matrix, an edge dictionary over its vertices (every vertex listed) or a Graph."""
    if form == "adjacency":
        return [A]
    d = {i: {int(j): 1.0 for j in np.nonzero(A[i])[0]} for i in range(A.shape[0])}
    if form == "dictionary":
        return [d]
    return Graph(d, {}, {}, "dictionary")
