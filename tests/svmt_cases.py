"""SvmTheta golden cases.  Every input is an adjacency matrix, stored in tests/golden/svm_theta.npz beside the
reference's results, so the tests need nothing but that file."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "svm_theta.npz")

# (name, constructor parameters) whose `fit` raises in the reference's `initialize`
ERROR_CASES = [("n_samples_zero", dict(n_samples=0)), ("n_samples_float", dict(n_samples=2.0)),
               ("range_list", dict(subsets_size_range=[2, 8])), ("range_decreasing", dict(subsets_size_range=(3, 2))),
               ("range_zero", dict(subsets_size_range=(0, 4))), ("range_short", dict(subsets_size_range=(2,))),
               ("range_float", dict(subsets_size_range=(2, 8.0))), ("metric_not_callable", dict(metric=5))]


def level_sum_metric(x, y):
    """A user metric over every level (the default one sees only the first)."""
    return float(np.sum(x) * np.sum(y))


def _rand_adj(rs, n, p, directed=False, lower=False, weights=None, loops=0):
    M = (rs.rand(n, n) < p).astype(float)
    if weights is not None:
        M *= rs.choice(weights, size=(n, n))
    if lower:
        A = np.tril(M, -1)
    elif directed:
        A = M - np.diag(np.diag(M))
    else:
        A = np.triu(M, 1)
        A = A + A.T
    for i in rs.choice(n, size=min(loops, n), replace=False):
        A[i, i] = 1.0
    return A


def _rand_set(seed, n_graphs, lo, hi, p=0.5, **kw):
    rs = np.random.RandomState(seed)
    return [_rand_adj(rs, int(rs.randint(lo, hi + 1)), p, **kw) for _ in range(n_graphs)]


def _drop(G, idx):
    return [A for i, A in enumerate(G) if i not in idx]


def cases(generate_dataset=None, mutag=None):
    """(name, X, Y or None, params): X and Y are lists of adjacency matrices.  `generate_dataset` (the reference's
    test generator) and `mutag` (MUTAG's adjacency matrices) are what the golden script passes; without them those
    cases are left out."""
    out = []
    if generate_dataset is not None:
        Xg, Yg = generate_dataset(n_graphs=100, r_vertices=(10, 20), r_connectivity=(0.4, 0.8), r_weight_edges=(1, 1),
                                  n_graphs_test=40, random_state=0, features="nl")
        adj = lambda G: [np.asarray(g[0], dtype=float) for g in G]
        out.append(("reference_tests", adj(Xg), adj(Yg), dict(random_state=0)))
    if mutag is not None:
        out.append(("mutag", mutag[:150], mutag[150:], dict(random_state=1)))
        out.append(("mutag_6_8", mutag[:150], mutag[150:], dict(random_state=1, subsets_size_range=(6, 8))))
    weights = np.array([0.0, 1e-11, 1e-10, 2e-10, -1.0, -1e-12, 0.5, 3.0])
    out += [
        ("small", _rand_set(2, 30, 2, 11), _rand_set(3, 10, 2, 11), dict(random_state=2)),
        # libsvm does not converge on some non-symmetric matrices (the reference then never returns): those are left out
        ("directed", _drop(_rand_set(4, 20, 3, 11, 0.4, directed=True), (10, 13)),
         _drop(_rand_set(5, 6, 3, 11, 0.4, directed=True), (2,)), dict(random_state=3)),
        ("lower_only", _rand_set(6, 10, 2, 11, 0.5, lower=True), _rand_set(7, 4, 2, 11, 0.5, lower=True),
         dict(random_state=4)),
        ("weights_loops", _drop(_rand_set(8, 16, 2, 11, 0.7, directed=True, weights=weights, loops=3), (3, 4, 14)),
         _rand_set(9, 6, 2, 11, 0.7, weights=weights, loops=2), dict(random_state=5)),
        ("empty", [np.zeros((n, n)) for n in (2, 3, 5, 8, 11, 12)], [np.zeros((4, 4))], dict(random_state=6)),
        ("range_6_8", _rand_set(10, 30, 6, 40, 0.3), _rand_set(11, 8, 6, 40, 0.3),
         dict(random_state=7, subsets_size_range=(6, 8))),
        ("levels_above_8", _rand_set(12, 20, 6, 16, 0.5), _rand_set(13, 5, 6, 16, 0.5),
         dict(random_state=8, n_samples=120, subsets_size_range=(3, 14))),
        ("one_sample", _rand_set(14, 12, 1, 9, 0.5), _rand_set(15, 4, 1, 9, 0.5),
         dict(random_state=9, n_samples=1, subsets_size_range=(1, 3))),
        ("many_samples", _rand_set(16, 10, 4, 9, 0.5), _rand_set(17, 3, 4, 9, 0.5),
         dict(random_state=10, n_samples=1000, subsets_size_range=(2, 4))),
        ("wide_range", _rand_set(18, 12, 2, 60, 0.2), _rand_set(19, 4, 2, 60, 0.2),
         dict(random_state=11, n_samples=300, subsets_size_range=(2, 70))),
    ]
    return out


# a second fit (the random stream continues), GraphKernel, a user metric: (name, base case, params)
SECOND_FIT = ("second_fit", "small", dict(random_state=12))
GRAPH_KERNEL = ("graph_kernel", "small", dict(kernel="SVMT", random_state=13))
GRAPH_KERNEL_DICT = ("graph_kernel_dict", "range_6_8",
                     dict(kernel={"name": "svm_theta", "subsets_size_range": (6, 8), "n_samples": 40},
                          random_state=14))
CUSTOM_METRIC = ("custom_metric", "levels_above_8",
                 dict(random_state=15, n_samples=120, subsets_size_range=(3, 14), metric=level_sum_metric))
# graphs of 5, 3, 1 and 6 vertices at subsets_size_range (2, 8): the third raises ZeroDivisionError after the draws of
# the first two
ZERO_DIVISION = ("zero_division", [np.ones((5, 5)) - np.eye(5), np.ones((3, 3)) - np.eye(3), np.zeros((1, 1)),
                                   np.zeros((6, 6))], dict(random_state=16))


def split(flat, sizes):
    """Square matrices of `sizes` from their concatenated row-major entries."""
    out, o = [], 0
    for n in sizes:
        out.append(flat[o:o + n * n].reshape(n, n))
        o += n * n
    return out


def load():
    """The golden file as a dict, with the inputs of every case unpacked: name -> (X, Y or None)."""
    z = dict(np.load(GOLDEN, allow_pickle=False))
    inputs = {}
    for key in z:
        if key.endswith("/x_sizes"):
            name = key[:-len("/x_sizes")]
            X = split(z[name + "/x_adj"], z[key])
            Y = split(z[name + "/y_adj"], z[name + "/y_sizes"]) if name + "/y_sizes" in z else None
            inputs[name] = (X, Y)
    return z, inputs
