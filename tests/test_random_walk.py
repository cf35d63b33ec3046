"""Host-side tests of RandomWalk / RandomWalkLabeled: the NumPy restatement against the reference's goldens,
parameter validation in the reference's order, the lamda tuning and its warnings, dispatch, the adjacency the
kernels read, the stacked eigen-solvers and pickling.  No GPU needed."""
import json
import os
import pickle
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import rw_oracle as O  # noqa: E402
from make_golden_random_walk import as_input, dict_inputs, unflat  # noqa: E402
from grakel_b200 import GraphKernel, RandomWalk, RandomWalkLabeled  # noqa: E402
from grakel_b200.kernels import _eigen_data, spectral_radii  # noqa: E402
from grakel_b200.packing import adjacency_and_labels  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "random_walk.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files if k != "dict" and not k.startswith("dict/")})


def case(name):
    meta = json.loads(str(GOLD[name + "/meta"]))
    X = unflat(GOLD[name + "/X_sizes"], GOLD[name + "/X_A"], GOLD[name + "/X_L"])
    Y = unflat(GOLD[name + "/Y_sizes"], GOLD[name + "/Y_A"], GOLD[name + "/Y_L"]) if name + "/Kt" in GOLD else None
    return meta, X, Y


@pytest.mark.parametrize("name", [c for c in CASES if json.loads(str(GOLD[c + "/meta"]))["params"].get("p") is None
                                  and json.loads(str(GOLD[c + "/meta"]))["params"].get("method_type", "fast") == "fast"
                                  and json.loads(str(GOLD[c + "/meta"]))["params"].get("kernel_type") is None])
def test_cg_oracle_matches_reference(name):
    meta, X, _ = case(name)
    K = GOLD[name + "/K"]
    lab = meta["cls"] == "RWL"
    for i in range(len(X)):
        for j in range(i, len(X)):
            (A, La), (B, Lb) = X[i], X[j]
            v, it = O.cg_pair(A, B, meta["lamda_used"], La if lab else None, Lb if lab else None)
            ref = K[i, j] if not meta["params"].get("normalize") else None
            if ref is not None:
                assert abs(v - ref) <= 1e-10 * abs(ref), (i, j, v, ref)
            assert 0 <= it <= 20


def test_series_and_spectral_oracle_match_reference():
    meta, X, _ = case("baseline_p")
    m = RandomWalk(**meta["params"])
    m.initialize()
    K = GOLD["baseline_p/K"]
    d = [O.series_pair(A, A, m.mu_)[0] for A, _ in X]
    for i in range(len(X)):
        for j in range(len(X)):
            s, mag = O.series_pair(X[min(i, j)][0], X[max(i, j)][0], m.mu_)
            assert abs(s / np.sqrt(d[i] * d[j]) - K[i, j]) <= 1e-12 * mag / np.sqrt(abs(d[i] * d[j]))
    meta, X, _ = case("fast_exponential_directed")
    K = GOLD["fast_exponential_directed/K"]
    qw = [O.eig_data(A) for A, _ in X]
    f = lambda z: np.exp(meta["lamda_used"] * z)
    d = [O.spectral_pair(q, w, q, w, f)[0] for q, w in qw]
    for i in range(len(X)):
        for j in range(i, len(X)):
            s, mag = O.spectral_pair(*qw[i], *qw[j], f)
            assert abs(s / np.sqrt(d[i] * d[j]) - K[i, j]) <= 1e-12 * mag / np.sqrt(abs(d[i] * d[j]))


def test_taylor_series_scaled_vector_on_hub_graphs():
    """The device's Taylor series restated: with M^k 1 and lamda^k / k! kept apart, M^k 1 overflows on a hub graph
    while lamda^k / k! underflows, their product is NaN and the series runs to its term cap; carrying the scaled vector
    lamda^k / k! M^k 1 sums every case to within 1e-11 of 1^T expm(lamda M) 1 (dense expm where kron(A, A) has at most
    3 600 rows, the eigh form above that)."""
    for name, A in O.hub_graphs().items():
        ref = O.expm_pair(A, A, 0.1) if A.shape[0] <= 60 else O.symmetric_expm_pair(A, A, 0.1)
        S, terms, capped = O.device_taylor(A, A, 0.1, scaled=True)
        assert not capped and abs(S - ref) <= 1e-11 * ref, (name, S, ref, terms)
        S0, _, capped0 = O.device_taylor(A, A, 0.1, scaled=False)
        if name == "K21":
            assert not capped0 and abs(S0 - ref) <= 1e-11 * ref
        else:
            assert capped0 and np.isnan(S0), name
    # the oracle's own series (taylor_pair) agrees with expm on a hub pair and on a labelled pair
    A, B = O.hub_graphs()["K21"], O.hub_graphs()["hub60"][:30, :30]
    assert abs(O.taylor_pair(A, B, 0.1) - O.expm_pair(A, B, 0.1)) <= 1e-11 * O.expm_pair(A, B, 0.1)
    La, Lb = [i % 3 for i in range(21)], [i % 2 for i in range(30)]
    ref = O.expm_pair(A, B, 0.1, La, Lb)
    assert abs(O.taylor_pair(A, B, 0.1, La, Lb) - ref) <= 1e-12 * ref


def test_validation_order_and_errors():
    with pytest.raises(ValueError, match="method_type"):
        RandomWalk(method_type="x", kernel_type="y").initialize()
    with pytest.raises(ValueError, match="kernel type"):
        RandomWalk(kernel_type="y").initialize()
    with pytest.raises(TypeError, match="lambda"):
        RandomWalk(lamda=0).initialize()
    with pytest.raises(TypeError, match="p must be"):
        RandomWalk(p=True).initialize()
    with pytest.raises(TypeError, match="p must be"):
        RandomWalk(p=0, lamda=-1).initialize()  # p is checked before lamda
    with pytest.raises(TypeError, match="p must be"):
        RandomWalkLabeled(p=2.0).initialize()
    k = RandomWalk(p=3, lamda=0.5, kernel_type="exponential")
    k.initialize()
    assert k.mu_ == [1, 0.5, 0.25 / 2, 0.125 / 6] and k._lamda == 0.5
    k = RandomWalk(p=2, lamda=0.5)
    k.initialize()
    assert k.mu_ == [1, 0.5, 0.25]


def test_tune_lamda_state_and_warnings():
    meta, X, _ = case("diverging_lamda")
    k = RandomWalk(**meta["params"])
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        k.fit(as_input(X))
    msgs = [str(x.message) for x in w if issubclass(x.category, RuntimeWarning)]
    assert msgs == meta["warnings"] and k._lamda == meta["lamda_used"] and k.lamda == 0.5
    lowered = k._lamda
    # a second fit on graphs that need no lowering keeps the lowered value
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        k.fit(as_input(X[:1]))
    assert k._lamda == lowered and not [x for x in w if issubclass(x.category, RuntimeWarning)]
    meta, X, Y = case("transform_larger_radius")
    k = RandomWalk(**meta["params"])
    k.fit(as_input(X))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        k._method_calling = 3
        k.parse_input(as_input(Y))
    assert [str(x.message) for x in w if issubclass(x.category, RuntimeWarning)] == meta["warnings"]


def test_negative_diagonal_warning_only_in_random_walk():
    with pytest.warns(RuntimeWarning, match="random walk kernels"):
        RandomWalk()._warn_unnormalizable(np.array([1.0, -2.0]))
    from grakel_b200 import VertexHistogram
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        VertexHistogram()._warn_unnormalizable(np.array([1.0, -2.0]))


def test_graph_kernel_points_to_the_estimators():
    for spec in ("RW", {"name": "random_walk", "with_labels": True}):
        with pytest.raises(NotImplementedError, match="RandomWalkLabeled"):
            GraphKernel(kernel=spec).initialize()
    with pytest.raises(NotImplementedError):
        RandomWalkLabeled(method_type="baseline")._route()


def test_adjacency_matches_reference():
    for i, g in enumerate(dict_inputs()):
        A, _ = adjacency_and_labels(g)
        assert np.array_equal(A, GOLD["dict/%d" % i]), i
    A = np.array([[0, -1, 0], [2, 1, 0], [0, 0, 0]])
    B, L = adjacency_and_labels(A, {0: "a", 1: "b", 2: "a"})
    assert np.array_equal(A, B) and B.dtype == np.float64 and L == ["a", "b", "a"]


def test_stacked_eig_is_bitwise_per_matrix():
    _, X, _ = case("fast_exponential_directed")
    mats = [A for A, _ in X] + [A for A, _ in case("mutag_rw_default")[1]]
    assert spectral_radii(mats) == [float(np.max(np.absolute(np.linalg.eigvals(A)))) for A in mats]
    q, w = _eigen_data(mats, False)
    ref = [O.eig_data(A) for A in mats]
    assert np.array_equal(q, np.concatenate([r[0] for r in ref])) and np.array_equal(w, np.concatenate([r[1] for r in ref]))
    sym = [A for A, _ in case("baseline_geometric_symmetric")[1]]
    q, w = _eigen_data(sym, True)
    ref = [np.linalg.eigh(A) for A in sym]
    assert np.array_equal(w, np.concatenate([r[0] for r in ref]))
    assert np.array_equal(q, np.concatenate([np.sum(r[1], axis=0) for r in ref]))


def test_pickles():
    _, X, _ = case("diverging_lamda")
    for cls in (RandomWalk, RandomWalkLabeled):
        k = cls(lamda=0.01, p=2)
        k.fit(as_input(X))
        k2 = pickle.loads(pickle.dumps(k))
        assert k2.mu_ == k.mu_ and k2._lamda == k._lamda and len(k2.X.mats) == len(X)
