"""GraphHopper on the CPU: the NumPy restatement (tests/gh_oracle.py) against the reference's goldens, and the
estimator's host-side behaviour (validation, weights, GraphKernel dispatch, pickling)."""
import os
import pickle
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from gh_oracle import GraphHopperOracle, adjacency_of, diameter, node_maps  # noqa: E402
from make_golden_graph_hopper import KERNEL_TYPES, _tag, cuneiform, inputs  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "graph_hopper.npz"))


def _close(K, R, kt):
    """1e-9 relative to the matrix scale (1e-6 for bridge) on the reference's finite entries: the reference's bridge
    takes sqrt of a difference of Gram entries (graph_hopper.py:368-383) and can give NaN on self similarities."""
    tol = 1e-6 if kt == "bridge" else 1e-9
    fin = np.isfinite(R)
    scale = max(np.max(np.abs(R[fin])), 1e-300)
    assert np.all(np.abs(K[fin] - R[fin]) <= tol * scale), np.max(np.abs(K[fin] - R[fin])) / scale


@pytest.mark.parametrize("name", ["sym", "sym_long", "dir"])
def test_oracle_node_maps_match_reference(name):
    X, _ = inputs()[name]
    delta = max(diameter(adjacency_of(x)[0]) for x in X) + 1
    for g in range(3):
        M = node_maps(adjacency_of(X[g])[0], delta)
        assert np.array_equal(M, GOLD["%s__M%d" % (name, g)])


@pytest.mark.parametrize("kt", KERNEL_TYPES, ids=_tag)
@pytest.mark.parametrize("name", ["sym", "sym_long", "dir"])
@pytest.mark.parametrize("norm", [False, True])
def test_oracle_gram_matches_reference(name, kt, norm):
    X, Y = inputs()[name]
    o = GraphHopperOracle(kt, normalize=norm)
    key = "%s__%s__%d" % (name, _tag(kt), int(norm))
    _close(o.fit_transform(X), GOLD[key + "__fit"], kt)
    _close(o.transform(Y), GOLD[key + "__tr"], kt)


@pytest.mark.parametrize("kt", KERNEL_TYPES, ids=_tag)
def test_oracle_cuneiform_matches_reference(kt):
    graphs = cuneiform()
    X = [graphs[i] for i in GOLD["cuneiform__idx"]]
    X = [[_adjacency(g, len(L)), L] for g, L in ((x[0], _relabel(x[1])) for x in X)]
    _close(GraphHopperOracle(kt).fit_transform(X), GOLD["cuneiform__" + _tag(kt)], kt)


def _relabel(L):
    keys = sorted(L)
    return {i: L[k] for i, k in enumerate(keys)}


def _adjacency(g, n):
    """Dense adjacency of an edge collection over vertex symbols 1..n of a TU graph (sorted order)."""
    edges = list(g.keys()) if isinstance(g, dict) else list(g)
    syms = sorted({x for e in edges for x in e})
    loc = {s: i for i, s in enumerate(syms)}
    A = np.zeros((n, n))
    for a, b in edges:
        A[loc[a], loc[b]] = 1
    return A


# ---------------------------------------------------------------- estimator (host side)
def test_kernel_type_validation():
    from grakel_b200 import GraphHopper
    X = inputs()["sym"][0]
    with pytest.raises(ValueError, match='Unsupported kernel with name "foo"'):
        GraphHopper(kernel_type="foo").fit(X)
    for bad in (3, ("gaussian",), ("gaussian", "x"), ("linear", 1.0)):
        with pytest.raises(TypeError, match="Unrecognized"):
            GraphHopper(kernel_type=bad).fit(X)


def test_scalar_and_ragged_labels_raise_type_error():
    from grakel_b200 import GraphHopper
    A = np.ones((3, 3)) - np.eye(3)
    with pytest.raises(TypeError, match="continuous node attributes"):
        GraphHopper().fit_transform([[A, {0: 1, 1: 2, 2: 3}]])
    with pytest.raises((TypeError, ValueError)):
        GraphHopper().fit_transform([[A, {0: [1.0, 2.0], 1: [1.0], 2: [0.0, 0.0]}]])
    with pytest.raises(TypeError, match="each element of X"):
        GraphHopper().fit_transform([[A]])


def test_weights_other_than_one_are_not_implemented():
    from grakel_b200 import GraphHopper
    A = np.array([[0, 2.0, 0], [2.0, 0, 1], [0, 1, 0]])
    with pytest.raises(NotImplementedError, match="edge weights"):
        GraphHopper().fit_transform([[A, {i: [float(i)] for i in range(3)}]])


def test_graph_kernel_dispatch():
    from grakel_b200 import GraphHopper, GraphKernel
    for name in ("GH", "graph_hopper"):
        gk = GraphKernel(kernel={"name": name, "kernel_type": "bridge"})
        cls, params = gk.make_kernel_([{"name": name, "kernel_type": "bridge"}], {})
        assert cls is GraphHopper and params == {"kernel_type": "bridge"}
    with pytest.raises(NotImplementedError):
        GraphKernel(kernel="random_walk").make_kernel_(["random_walk"], {})


@pytest.mark.parametrize("kt", ["linear", ("gaussian", 0.5), "bridge"], ids=str)
def test_initialized_estimator_pickles(kt):
    from grakel_b200 import GraphHopper
    gh = GraphHopper(kernel_type=kt)
    gh.initialize()
    gh._max_diam = 4
    gh2 = pickle.loads(pickle.dumps(gh))
    assert gh2.kernel_type == kt and gh2._max_diam == 4 and gh2.calculate_norm_ == gh.calculate_norm_
    x = (np.ones((2, 4)), np.array([[0.0, 1.0], [1.0, 0.5]]))
    assert gh2.metric_(x, x) == gh.metric_(x, x)
