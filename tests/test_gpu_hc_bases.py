"""HadamardCode over SubgraphMatching, PyramidMatch and NeighborhoodSubgraphPairwiseDistance on the device: == against
the real reference's goldens, and HadamardCode over SubgraphMatching (one clique enumeration for every level) bit for
bit against the per-level device route -- n_iter SubgraphMatching runs on the level's Hadamard-code classes, summed in
level order -- at the benchmark's scale."""
import contextlib
import os
import sys

import numpy as np
import pytest

import hc_bases_cases as cases
import hc_bases_oracle as oracle
import hc_oracle
from grakel_b200 import (GraphKernel, HadamardCode, NeighborhoodSubgraphPairwiseDistance, PyramidMatch,
                         SubgraphMatching, _lib)

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "hc_bases.npz"))
BASES = {"SM": SubgraphMatching, "PM": PyramidMatch, "NSPD": NeighborhoodSubgraphPairwiseDistance}
RUNS = [(name, n_iter) for name, (_, _, _, _, n_iters) in sorted(cases.cases().items())
        if name not in cases.GRAPH_OBJECT_CASES for n_iter in n_iters]


def hc(base, params, n_iter, normalize=False):
    return HadamardCode(n_iter=n_iter, normalize=normalize, base_graph_kernel=(BASES[base], dict(params)))


@pytest.mark.parametrize("name,n_iter", RUNS)
def test_goldens(name, n_iter):
    base, X, Ys, params, _ = cases.cases()[name]
    for norm in (False, True):
        key = "%s_%d%s" % (name, n_iter, "_norm" if norm else "")
        k = hc(base, params, n_iter, norm)
        np.testing.assert_array_equal(k.fit_transform(X), G[key + "_fit_transform"])
        np.testing.assert_array_equal(k.diagonal(), G[key + "_ft_diag"])
        for t, Y in sorted(Ys.items()):
            k = hc(base, params, n_iter, norm)
            k.fit_transform(X)
            np.testing.assert_array_equal(k.transform(Y), G["%s_%s_ft_transform" % (key, t)])
            k = hc(base, params, n_iter, norm)
            np.testing.assert_array_equal(k.fit(X).transform(Y), G["%s_%s_fit_transform_y" % (key, t)])
            xd, yd = k.diagonal()
            np.testing.assert_array_equal(xd, G["%s_%s_fit_diag_x" % (key, t)])
            np.testing.assert_array_equal(yd, G["%s_%s_fit_diag_y" % (key, t)])


def ke_real(a, b):
    """Real weights that are not exact in binary: every summation order shows in the bits."""
    return 0.7 if a == b else 0.1


def bench_workload(n):
    from bench import gen_list
    return [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in gen_list(n, 40, 0)]


def per_level(params, n_iter, X):
    """The per-level device route: one SubgraphMatching (sm_pairs) per level on the level's Hadamard-code classes as
    vertex labels, K summed in level order."""
    enum = hc_oracle.enumerate_labels([x[1] for x in X])
    Ks = []
    for lx in oracle.level_elements(X, n_iter, enum):
        Ks.append(SubgraphMatching(**params).fit_transform(lx))
    return np.sum(Ks, axis=0)


@pytest.mark.parametrize("params", [{"k": 3}, {"k": 3, "ke": ke_real}, {"k": 5}, {"k": 5, "ke": ke_real}])
def test_bench_scale_equals_the_per_level_route(params):
    """bench.gen_list(2000, 40, 0) with edge labels (L_u + L_v) % 3, n_iter = 5: the one-pass K equals the level sum
    of five sm_pairs runs bit for bit, with exact (integer) and real (ke_real) sums."""
    X = bench_workload(2000)
    np.testing.assert_array_equal(hc("SM", params, 5).fit_transform(X), per_level(params, 5, X))


@pytest.mark.parametrize("params", [{"k": 4}, {"k": 4, "ke": ke_real}])
def test_row_ranges_and_device_output(params, monkeypatch):
    """Row ranges, device output and the global-record route give the host K."""
    X = bench_workload(300)
    Xf, Y = X[:220], X[220:]
    k = hc("SM", params, 3)
    K = k.fit_transform(Xf)
    Kt = k.transform(Y)
    Kr, _, _ = k._run(k.X, len(Xf), k._width, row_range=(7, 131))
    np.testing.assert_array_equal(Kr, K[7:131])
    import torch
    dev = torch.zeros((len(Xf), len(Xf)), dtype=torch.float64, device="cuda")
    k._run(k.X, len(Xf), k._width, device_ptr=dev.data_ptr())
    torch.cuda.synchronize()
    np.testing.assert_array_equal(dev.cpu().numpy(), K)
    monkeypatch.setenv("GRAKEL_B200_SM_GLOBAL", "1")
    np.testing.assert_array_equal(hc("SM", params, 3).fit_transform(Xf), K)
    np.testing.assert_array_equal(hc("SM", params, 3).fit(Xf).transform(Y), Kt)


def test_bin_cap_refuses_before_any_launch():
    """n_iter * min(k, largest graph) may be 64: k = 4 on graphs of 4 or more vertices allows n_iter = 16."""
    X = bench_workload(12)
    p = {"k": 4}
    np.testing.assert_array_equal(hc("SM", p, 16).fit_transform(X), per_level(p, 16, X))
    k = hc("SM", p, 17)
    k.fit(X)
    data = k.X.base
    sm = k._sm
    gp, rp, ci, lab, elids, _, et, flags = sm._pack([(n, e, [0] * n, el) for n, e, _, el in data.graphs])
    with _lib.engine() as eng:
        eng.pack(gp, rp, ci, lab, None, None)
        with pytest.raises(NotImplementedError, match="more than 64"):
            eng.sm_hc_features(4, 17, np.zeros((len(lab), 17), dtype=np.int32), sm.lambdas_, et, elids, flags)
    with pytest.raises(NotImplementedError, match="more than 64"):
        k.fit_transform(X)


def test_live_bytes_return_after_close(monkeypatch):
    before = _lib.live_bytes()
    eng = _lib.Engine()
    monkeypatch.setattr(_lib, "engine", lambda device=None: contextlib.nullcontext(eng))
    try:
        X = cases.fit_set()
        Y = cases.transform_same()
        for base, p in (("SM", {"k": 4}), ("SM", {"k": 3, "ke": ke_real}), ("PM", {}), ("NSPD", {"r": 1, "d": 2})):
            k = hc(base, p, 3)
            k.fit_transform(X)
            k.transform(Y)
        assert _lib.live_bytes()[0] > before[0]
    finally:
        eng.close()
    assert _lib.live_bytes() == before


def test_dist_is_refused():
    k = hc("SM", {}, 2).fit(cases.fit_set())
    sm, data = k._sm, k.X.base
    gp, rp, ci, _, elids, _, et, flags = sm._pack(data.graphs)
    with _lib.engine() as eng:
        eng.pack(gp, rp, ci, None, None, None)
        eng.sm_hc_features(5, 2, None, sm.lambdas_, et, elids, _lib.GK_SM_KV_NONE | (flags & ~3))
        with pytest.raises(NotImplementedError, match="GK_DIST"):
            eng.gram(len(data.graphs), dist=True)


def test_graph_kernel_dispatch():
    X = cases.fit_set()
    for base, name, p in (("SM", "SM", {"k": 3}), ("PM", "PM", {}), ("NSPD", "NSPD", {"r": 1, "d": 2})):
        K = hc(base, p, 2).fit_transform(X)
        spec = [{"name": "HC", "n_iter": 2}, dict(name=name, **p)]
        np.testing.assert_array_equal(GraphKernel(kernel=spec).fit_transform(X), K)
