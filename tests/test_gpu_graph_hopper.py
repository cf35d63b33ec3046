"""GraphHopper on the H100 (run with -m gpu): device node maps against the NumPy restatement bit for bit, the three
node kernels against it and against the reference's goldens, transform / normalise / row blocks, determinism and
exact symmetry of the node-pair Gram, and the callable route."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from gh_oracle import GraphHopperOracle, adjacency_of, diameter, node_maps  # noqa: E402
from make_golden_graph_hopper import KERNEL_TYPES, _tag, connected, directed, inputs, paths  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(HERE, "golden", "graph_hopper.npz"))


def _rel(K, R):
    return np.max(np.abs(K - R)) / max(np.max(np.abs(R)), 1e-300)


def _device_maps(X):
    from grakel_b200 import _lib
    from grakel_b200.packing import pack
    b = pack(X, "sp", need_labels=True, len_ok=lambda n: n >= 2, attributes=True)
    with _lib.engine() as eng:
        eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, None, None, b.attrs)
        st = eng.gh_features(_lib.GK_GH_LINEAR)
        gp = b.graph_ptr
        return [eng.gh_node_maps(g, int(gp[g + 1] - gp[g])) for g in range(b.n_graphs)], st


def _with_isolated(N, seed):
    """ER graphs with isolated vertices, single-vertex graphs and directed sinks."""
    rs = np.random.RandomState(seed)
    X = []
    for k in range(N):
        n = 1 if k % 5 == 0 else int(rs.randint(3, 12))
        A = (rs.rand(n, n) < 1.5 / n).astype(float)
        np.fill_diagonal(A, 0)
        X.append([A, {i: rs.rand(2).round(3).tolist() for i in range(n)}])
    return X


def _big():
    """A 200-vertex chorded cycle, whose working set (delta near 100) is above the shared-memory limit of the node-map
    kernel, plus small graphs that stay in shared memory."""
    rs = np.random.RandomState(7)
    n = 200
    A = np.zeros((n, n))
    A[np.arange(n), (np.arange(n) + 1) % n] = 1
    for _ in range(3):
        a, b = rs.randint(n, size=2)
        if a != b:
            A[a, b] = 1
    A = np.maximum(A, A.T)
    return [[A, {i: rs.rand(2).round(3).tolist() for i in range(n)}]] + connected(3, 8, 8, dim=2)


CASES = {
    "sym": lambda: connected(20, 10, 11),
    "dir": lambda: directed(20, 9, 12),
    "isolated": lambda: _with_isolated(25, 13),
    "long": lambda: paths(3, 45, 14),
}


@pytest.mark.parametrize("case", list(CASES))
def test_node_maps_bit_exact(case):
    X = CASES[case]()
    maps, st = _device_maps(X)
    delta = max(diameter(adjacency_of(x)[0]) for x in X) + 1
    assert st.level_dims[0] == delta
    if case == "long":
        assert delta > 40
    for x, M in zip(X, maps):
        assert np.array_equal(M, node_maps(adjacency_of(x)[0], delta))


def test_node_maps_global_workspace():
    X = _big()
    maps, st = _device_maps(X)
    delta = int(st.level_dims[0])
    assert 200 * (delta + 1) * 8 > 96 * 1024  # the 200-vertex graph runs from the global workspace
    for x, M in zip(X, maps):
        assert np.array_equal(M, node_maps(adjacency_of(x)[0], delta))


@pytest.mark.parametrize("case", ["sym", "dir", "isolated"])
@pytest.mark.parametrize("kt", KERNEL_TYPES, ids=_tag)
def test_gram_against_oracle(case, kt):
    from grakel_b200 import GraphHopper
    X = CASES[case]()
    gh = GraphHopper(kernel_type=kt)
    K = gh.fit_transform(X)
    R = GraphHopperOracle(kt).fit_transform(X)
    if kt == "linear":
        assert gh.stats_.gram_path == 4
        assert _rel(K, R) <= 1e-5
    else:
        assert gh.stats_.gram_path == 6
        assert _rel(K, R) <= 1e-9
        assert np.array_equal(K, K.T)


def test_linear_mixed_sign_takes_fp64():
    from grakel_b200 import GraphHopper
    X = connected(30, 10, 21)
    for _A, L in X:
        for v in L:
            L[v] = [a - 0.5 for a in L[v]]
    gh = GraphHopper()
    K = gh.fit_transform(X)
    assert gh.stats_.gram_path == 5
    assert _rel(K, GraphHopperOracle("linear").fit_transform(X)) <= 1e-9


@pytest.mark.parametrize("name", ["sym", "sym_long", "dir"])
@pytest.mark.parametrize("kt", KERNEL_TYPES, ids=_tag)
@pytest.mark.parametrize("norm", [False, True])
def test_goldens(name, kt, norm):
    from grakel_b200 import GraphHopper
    X, Y = inputs()[name]
    key = "%s__%s__%d" % (name, _tag(kt), int(norm))
    gh = GraphHopper(kernel_type=kt, normalize=norm)
    tol = 1e-5 if kt == "linear" else (1e-6 if kt == "bridge" else 1e-9)
    for K, R in ((gh.fit_transform(X), GOLD[key + "__fit"]), (gh.transform(Y), GOLD[key + "__tr"])):
        fin = np.isfinite(R)
        assert K.shape == R.shape
        assert np.max(np.abs(K[fin] - R[fin])) <= tol * np.max(np.abs(R[fin]))


@pytest.mark.parametrize("kt", ["gaussian", "bridge"])
def test_transform_normalize_rows_and_determinism(kt):
    from grakel_b200 import GraphHopper, _lib
    from grakel_b200.packing import pack
    X, Y = connected(70, 12, 31), paths(5, 20, 32)
    o = GraphHopperOracle(kt, normalize=True)
    Ro = o.fit_transform(X)
    gh = GraphHopper(kernel_type=kt, normalize=True)
    K = gh.fit_transform(X)
    assert _rel(K, Ro) <= 1e-9 and np.array_equal(K, K.T)
    Ky = gh.transform(Y)
    assert _rel(Ky, o.transform(Y)) <= 1e-9
    # row blocks equal the full matrix's rows bit for bit; two runs are bit-identical
    b = pack(X, "sp", need_labels=True, len_ok=lambda n: n >= 2, attributes=True)
    nk = _lib.GK_GH_GAUSSIAN if kt == "gaussian" else _lib.GK_GH_BRIDGE
    with _lib.engine() as eng:
        eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, None, None, b.attrs)
        eng.gh_features(nk, 1.0)
        full, _, _ = eng.gram(b.n_graphs)
        again, _, _ = eng.gram(b.n_graphs)
        blk, _, _ = eng.gram(b.n_graphs, row_range=(17, 53))
    assert np.array_equal(full, again)
    assert np.array_equal(blk, full[17:53])
    assert np.array_equal(full, full.T)


def test_callable_route_agrees_with_linear():
    from grakel_b200 import GraphHopper

    def linear_kernel(x, y):
        M_i, NA_i = x
        M_j, NA_j = y
        return np.dot(np.dot(M_i, M_j.T).flat, np.dot(NA_i, NA_j.T).flat)

    X, Y = inputs()["sym_long"]
    a, b = GraphHopper(kernel_type=linear_kernel), GraphHopper(kernel_type="linear")
    assert _rel(a.fit_transform(X), b.fit_transform(X)) <= 1e-5
    assert _rel(a.transform(Y), b.transform(Y)) <= 1e-5
    assert a._max_diam == b._max_diam


def test_fitted_estimator_pickles():
    import pickle
    from grakel_b200 import GraphHopper
    X, Y = inputs()["sym"]
    gh = GraphHopper(kernel_type=("gaussian", 0.3)).fit(X)
    gh2 = pickle.loads(pickle.dumps(gh))
    assert np.array_equal(gh.transform(Y), gh2.transform(Y))
