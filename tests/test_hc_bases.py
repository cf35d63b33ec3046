"""HadamardCode over SubgraphMatching, PyramidMatch and NeighborhoodSubgraphPairwiseDistance on the host: the in-repo
restatement (tests/hc_bases_oracle.py) against the real reference's goldens (tests/golden/make_golden_hc_bases.py),
the dispatch, and the refusals, all raised before any device work."""
import os

import numpy as np
import pytest

import hc_bases_cases as cases
import hc_bases_oracle as oracle
from grakel_b200 import (Graph, GraphKernel, HadamardCode, NeighborhoodSubgraphPairwiseDistance, OddSth,
                         PyramidMatch, SubgraphMatching)
from grakel_b200.packing import Block

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "hc_bases.npz"))
BASES = {"SM": SubgraphMatching, "PM": PyramidMatch, "NSPD": NeighborhoodSubgraphPairwiseDistance}
RUNS = [(name, n_iter) for name, (base, _, _, _, n_iters) in sorted(cases.cases().items())
        if base != "PM" and name not in cases.GRAPH_OBJECT_CASES for n_iter in n_iters]


def hc(base, params, n_iter=2, normalize=False):
    return HadamardCode(n_iter=n_iter, normalize=normalize, base_graph_kernel=(BASES[base], dict(params)))


@pytest.mark.parametrize("name,n_iter", RUNS)
def test_restatement_matches_the_reference(name, n_iter):
    base, X, Ys, params, _ = cases.cases()[name]
    key = "%s_%d" % (name, n_iter)
    if base == "SM":
        assert np.array_equal(oracle.sm_kernel(params, n_iter, X), G[key + "_fit_transform"])
        assert np.array_equal(oracle.sm_kernel(params, n_iter, X, normalize=True), G[key + "_norm_fit_transform"])
    else:
        assert np.array_equal(oracle.nspd_kernel(params, n_iter, X), G[key + "_fit_transform"])
    for t, Y in Ys.items():
        if base == "SM":
            K = oracle.sm_kernel(params, n_iter, X, Y)
            assert np.array_equal(oracle.sm_kernel(params, n_iter, X, Y, normalize=True),
                                  G["%s_norm_%s_fit_transform_y" % (key, t)])
        else:
            K = oracle.nspd_kernel(params, n_iter, X, Y)
        assert np.array_equal(K, G["%s_%s_fit_transform_y" % (key, t)])
        assert np.array_equal(K, G["%s_%s_ft_transform" % (key, t)])
        if t == "wide" and (base != "SM" or params.get("kv", 0) is not None):
            assert not K.any()  # the widened vectors share no label with the fitted ones


@pytest.mark.parametrize("name", sorted(cases.error_cases()))
def test_reference_errors(name):
    """The element checks run at parse time, before any relabelling or pair reaches the device."""
    base, X, params = cases.error_cases()[name]
    etype, msg = G["err_%s_error" % name]
    with pytest.raises(Exception) as e:
        hc(base, params).fit_transform(X)
    assert type(e.value).__name__ == etype and str(e.value) == msg


def test_graph_objects_are_refused_like_the_reference():
    X = [Graph(*x) for x in cases.fit_set()]
    etype, msg = G["sm_graph_objects_2_fit_transform_error"]
    for base in BASES:
        with pytest.raises(ValueError) as e:
            hc(base, {}).fit(X)
        assert type(e.value).__name__ == etype and str(e.value) == msg


def test_custom_vertex_kernel_is_refused_at_fit():
    with pytest.raises(NotImplementedError, match="kv=_dirac or kv=None"):
        hc("SM", {"kv": lambda a, b: 1}).fit(cases.fit_set())


def test_base_kernel_arguments_are_checked_at_fit():
    X = cases.fit_set()
    with pytest.raises(TypeError, match="lw can either"):
        hc("SM", {"lw": "flat"}).fit(X)
    with pytest.raises(TypeError, match="with labels must be a boolean"):
        hc("PM", {"with_labels": 1}).fit(X)
    with pytest.raises(ValueError, match="r must be a positive integer"):
        hc("NSPD", {"r": -1}).fit(X)


@pytest.mark.parametrize("base", sorted(BASES))
def test_packed_block_is_refused(base):
    b = Block([0, 2], [0, 1, 2], [1, 0], None, [0, 1])
    b.mode = "wl"
    with pytest.raises(NotImplementedError, match="pass the list of graphs"):
        hc(base, {}).fit(b)


def test_odd_sth_stays_refused():
    with pytest.raises(NotImplementedError, match="outside the device hot path"):
        HadamardCode(base_graph_kernel=OddSth).fit(cases.fit_set())


@pytest.mark.parametrize("spec,base", [
    (["HC", "SM"], SubgraphMatching), (["HC", "PM"], PyramidMatch),
    (["HC", "NSPD"], NeighborhoodSubgraphPairwiseDistance),
    ([{"name": "HC", "n_iter": 2}, {"name": "SM", "k": 3}], SubgraphMatching),
    ([{"name": "hadamard_code"}, {"name": "pyramid_match", "with_labels": False}], PyramidMatch),
    ([{"name": "hadamard_code"}, {"name": "neighborhood_subgraph_pairwise_distance", "r": 1}],
     NeighborhoodSubgraphPairwiseDistance)])
def test_graph_kernel_spells_hc_over_the_new_bases(spec, base):
    gk = GraphKernel(kernel=spec)
    gk.initialize()
    k = gk.kernel_
    assert isinstance(k, HadamardCode)
    k.initialize()
    assert k.base_graph_kernel_[0] is base
