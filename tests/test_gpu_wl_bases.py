"""WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance and OddSth on the device: == against the real
reference's goldens and against the in-repo restatement (tests/wl_bases_oracle.py) at the benchmark's graph sizes."""
import os
import sys

import numpy as np
import pytest

import wl_bases_cases as cases
import wl_bases_oracle as oracle
from grakel_b200 import GraphKernel, NeighborhoodSubgraphPairwiseDistance, OddSth, WeisfeilerLehman
from grakel_b200.kernels import Fitted

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "wl_bases.npz"))
KINDS = {"NSPD": NeighborhoodSubgraphPairwiseDistance, "ODD": OddSth}


def wl(kind, params, n_iter, normalize=False):
    return WeisfeilerLehman(n_iter=n_iter, normalize=normalize, base_graph_kernel=(KINDS[kind], dict(params)))


@pytest.mark.parametrize("n_iter", cases.N_ITERS)
@pytest.mark.parametrize("name", sorted(cases.BASES))
def test_goldens(name, n_iter):
    kind, params = cases.BASES[name]
    X, Y = cases.fit_set(), cases.transform_set()
    for norm in (False, True):
        key = "%s_%d%s" % (name, n_iter, "_norm" if norm else "")
        k = wl(kind, params, n_iter, norm)
        K = k.fit_transform(X)
        assert np.array_equal(K, G[key + "_fit_transform"]), key
        assert np.array_equal(k.diagonal(), np.diagonal(G["%s_%d_fit_transform" % (name, n_iter)]))
        assert np.array_equal(k.transform(Y), G[key + "_ft_transform"]), key
        k = wl(kind, params, n_iter, norm).fit(X)
        if key + "_fit_transform_y_error" in G.files:
            etype, msg = G[key + "_fit_transform_y_error"]
            with pytest.raises(AttributeError, match="_phi_X"):
                k.transform(Y)
            assert etype == "AttributeError"
        else:
            assert np.array_equal(k.transform(Y), G[key + "_fit_transform_y"]), key


def bench_workload(n):
    from bench import gen_list
    return [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in gen_list(n, 40, 0)]


@pytest.mark.parametrize("kind,params", [("NSPD", {}), ("ODD", {}), ("ODD", {"h": 2})])
def test_bench_graphs_at_n_iter_5(kind, params):
    """bench.gen_list(2000, 40, 0) graphs (the tools/bench_nspd.py workload), n_iter = 5.  A fit_transform and a
    transform against the restatement, on as many graphs as its cost allows (the NSPD restatement takes about a second
    per graph and level at r = 3, d = 4), then all 2000 graphs on the device: symmetric, and for OddSth without a hash
    retry."""
    X = bench_workload(2000)
    nf, nt = (3, 1) if kind == "NSPD" else (200, 60)
    Xf, Y = X[:nf], X[nf:nf + nt]
    k = wl(kind, params, 5)
    assert np.array_equal(k.fit_transform(Xf), oracle.kernel(kind, params, 5, Xf))
    assert np.array_equal(k.transform(Y), oracle.kernel(kind, params, 5, Xf, Y))
    k = wl(kind, params, 5)
    K = k.fit_transform(X)
    assert K.shape == (2000, 2000) and np.array_equal(K, K.T) and np.all(np.isfinite(K))
    if kind == "ODD":
        assert k.stats_.hash_retries == 0


def test_nspd_64_levels_at_n_iter_5():
    X, Y = cases.fit_set(), cases.transform_set()
    p = {"r": 7, "d": 7}
    k = wl("NSPD", p, 5)
    assert np.array_equal(k.fit_transform(X), oracle.kernel("NSPD", p, 5, X))
    assert np.array_equal(k.transform(Y), oracle.kernel("NSPD", p, 5, X, Y))


@pytest.mark.parametrize("kind,params", [("NSPD", {"r": 1, "d": 2}), ("ODD", {})])
def test_frozen_deep_levels(kind, params):
    """Many small graphs: the deep WL levels change few vertices, so the relabel hands on sparse ids."""
    X = cases.graphs(300, 6, 11)
    Y = cases.graphs(40, 6, 12, new_labels=True)
    k = wl(kind, params, 5)
    assert np.array_equal(k.fit_transform(X), oracle.kernel(kind, params, 5, X))
    assert np.array_equal(k.transform(Y), oracle.kernel(kind, params, 5, X, Y))


@pytest.mark.parametrize("kind,params", [("NSPD", {"r": 1, "d": 2}), ("ODD", {"h": 2})])
def test_transform_row_range_from_joint_input(kind, params):
    X, Y = cases.fit_set(), cases.transform_set()
    k = wl(kind, params, 2).fit(X)
    K = k.transform(Y)
    Kr, _, _ = k._base_run(Fitted.concat(k.X, k.parse_input(Y)), k._nx, row_range=(1, 3))
    assert np.array_equal(Kr, K[1:3])


def test_graph_kernel_dispatch():
    X = cases.fit_set()
    for spec, kind, params in [({"name": "NSPD", "r": 1, "d": 2}, "NSPD", {"r": 1, "d": 2}),
                               ({"name": "ODD", "h": 2}, "ODD", {"h": 2}),
                               ({"name": "odd_sth"}, "ODD", {})]:
        gk = GraphKernel(kernel=[{"name": "WL", "n_iter": 2}, spec])
        assert np.array_equal(gk.fit_transform(X), G["%s_2_fit_transform" % {
            ("NSPD", 1): "nspd12", ("ODD", 2): "odd2", ("ODD", None): "oddN"}[(kind, params.get("r", params.get("h")))]])


def test_oddsth_refusals_before_allocation():
    """More than 4096 vertices in a graph, and 2^30 or more (root, vertex) pairs over the n_iter + 1 levels."""
    def ring(n):
        g = {}
        for v in range(n):
            g[(v, (v + 1) % n)] = 1
            g[((v + 1) % n, v)] = 1
        return [g, {v: v % 3 for v in range(n)}]
    with pytest.raises(NotImplementedError, match="4096"):
        wl("ODD", {}, 1).fit_transform([ring(4097)])
    # 11 graphs of 4096 vertices: 1.85e8 pairs per level, 1.1e9 over 6 levels (1.6e8 over 1: the single level fits)
    with pytest.raises(NotImplementedError, match="2\\^30"):
        wl("ODD", {}, 5).fit_transform([ring(4096) for _ in range(11)])
