"""WeisfeilerLehman over SubgraphMatching on the host: the in-repo restatement (tests/wl_sm_oracle.py) against the real
reference's goldens (tests/golden/make_golden_wl_sm.py), and the estimator's checks and refusals, all raised before
any device work."""
import os

import numpy as np
import pytest

import wl_sm_cases as cases
import wl_sm_oracle as oracle
from grakel_b200 import Graph, GraphKernel, SubgraphMatching, WeisfeilerLehman
from grakel_b200.packing import Block

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "wl_sm.npz"))
RUNS = [(name, n_iter) for name, (_, _, _, n_iters) in sorted(cases.cases().items()) for n_iter in n_iters]


def wl(params, n_iter=2, normalize=False):
    return WeisfeilerLehman(n_iter=n_iter, normalize=normalize, base_graph_kernel=(SubgraphMatching, dict(params)))


@pytest.mark.parametrize("name,n_iter", RUNS)
def test_restatement_matches_the_reference(name, n_iter):
    X, Y, params, _ = cases.cases()[name]
    key = "%s_%d" % (name, n_iter)
    K = oracle.kernel(params, n_iter, X)
    assert np.array_equal(K, G[key + "_fit_transform"])
    assert np.array_equal(np.diagonal(K), G[key + "_ft_diag"])
    assert np.array_equal(oracle.kernel(params, n_iter, X, normalize=True), G[key + "_norm_fit_transform"])
    Ky = oracle.kernel(params, n_iter, X, Y)
    assert np.array_equal(Ky, G[key + "_ft_transform"])
    assert np.array_equal(Ky, G[key + "_fit_transform_y"])
    Kn = oracle.kernel(params, n_iter, X, Y, normalize=True)
    assert np.array_equal(Kn, G[key + "_norm_ft_transform"])
    assert np.array_equal(Kn, G[key + "_norm_fit_transform_y"])


@pytest.mark.parametrize("name", sorted(cases.error_cases()))
def test_reference_errors(name):
    """The element checks run at parse time, before the WL partition or any pair reaches the device."""
    X, params = cases.error_cases()[name]
    etype, msg = G["err_%s_error" % name]
    with pytest.raises(Exception) as e:
        wl(params).fit_transform(X)
    assert type(e.value).__name__ == etype and str(e.value) == msg


def test_graph_object_without_edge_labels_is_refused_like_the_reference():
    X = [Graph(x[0], x[1]) for x in cases.fit_set()]
    etype, msg = G["err_no_edge_labels_error"]
    with pytest.raises(TypeError) as e:
        wl({}).fit(X)
    assert str(e.value) == msg


def test_custom_vertex_kernel_is_refused_at_fit():
    with pytest.raises(NotImplementedError, match="kv=_dirac or kv=None"):
        wl({"kv": lambda a, b: 1}).fit(cases.fit_set())


def test_base_kernel_arguments_are_checked_at_fit():
    X = cases.fit_set()
    with pytest.raises(TypeError, match="kv must be callable"):
        wl({"kv": 3}).fit(X)
    with pytest.raises(TypeError, match="lw can either"):
        wl({"lw": "flat"}).fit(X)
    with pytest.raises(NotImplementedError, match="k < 0"):
        wl({"k": -1}).fit(X)


def test_packed_block_is_refused():
    b = Block([0, 2], [0, 1, 2], [1, 0], None, [0, 1])
    b.mode = "wl"
    with pytest.raises(NotImplementedError, match="edge dictionary"):
        wl({}).fit(b)


@pytest.mark.parametrize("spec", [["WL", "SM"], [{"name": "WL", "n_iter": 2}, {"name": "SM", "k": 3}],
                                  [{"name": "weisfeiler_lehman"}, {"name": "subgraph_matching"}]])
def test_graph_kernel_spells_wl_over_sm(spec):
    gk = GraphKernel(kernel=spec)
    gk.initialize()
    k = gk.kernel_
    assert isinstance(k, WeisfeilerLehman)
    k.initialize()
    assert k._base_graph_kernel is SubgraphMatching
