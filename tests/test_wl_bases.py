"""WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance and OddSth on the host: the in-repo restatement
(tests/wl_bases_oracle.py) against the real reference's goldens (tests/golden/make_golden_wl_bases.py), and the
estimator's argument checks."""
import os

import numpy as np
import pytest

import wl_bases_cases as cases
import wl_bases_oracle as oracle
from grakel_b200 import NeighborhoodSubgraphPairwiseDistance, OddSth, WeisfeilerLehman

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "wl_bases.npz"))


@pytest.mark.parametrize("n_iter", cases.N_ITERS)
@pytest.mark.parametrize("name", sorted(cases.BASES))
def test_restatement_matches_the_reference(name, n_iter):
    kind, params = cases.BASES[name]
    X, Y = cases.fit_set(), cases.transform_set()
    key = "%s_%d" % (name, n_iter)
    K = oracle.kernel(kind, params, n_iter, X)
    assert np.array_equal(K, G[key + "_fit_transform"])
    assert np.array_equal(oracle.normalized(K), G[key + "_norm_fit_transform"])
    Ky = oracle.kernel(kind, params, n_iter, X, Y)
    assert np.array_equal(Ky, G[key + "_ft_transform"])
    assert np.array_equal(Ky, G[key + "_fit_transform_y"])


def test_reference_raises_for_normalized_oddsth_transform_after_fit():
    for name, (kind, _) in cases.BASES.items():
        for n_iter in cases.N_ITERS:
            key = "%s_%d_norm_fit_transform_y" % (name, n_iter)
            if kind == "ODD":
                assert list(G[key + "_error"]) == ["AttributeError", "'OddSth' object has no attribute '_phi_X'"]
            else:
                assert key in G.files


def test_base_kernel_arguments_are_checked_at_fit():
    X = cases.fit_set()
    with pytest.raises(NotImplementedError, match="64"):
        WeisfeilerLehman(base_graph_kernel=(NeighborhoodSubgraphPairwiseDistance, {"r": 7, "d": 8})).fit(X)
    with pytest.raises(ValueError, match="r must be"):
        WeisfeilerLehman(base_graph_kernel=(NeighborhoodSubgraphPairwiseDistance, {"r": -1})).fit(X)
    with pytest.raises(ValueError, match="h must be"):
        WeisfeilerLehman(base_graph_kernel=(OddSth, {"h": 0})).fit(X)


def test_nspd_base_needs_edge_labels():
    X = [x[:2] for x in cases.fit_set()]
    with pytest.raises(TypeError):
        WeisfeilerLehman(base_graph_kernel=NeighborhoodSubgraphPairwiseDistance).fit(X)


def test_level_numbering_of_a_transform_continues_the_fit():
    """wl_reference_dictionaries with n_fit_vertices: classes the fitted vertices have keep their fit numbers."""
    X, Y = cases.fit_set(), cases.transform_set()
    fit_only = oracle.level_elements(X, None, 2)
    joint = oracle.level_elements(X, Y, 2)
    for (fx, _), (jx, jy) in zip(fit_only, joint):
        assert [e[1] for e in fx] == [e[1] for e in jx]
