"""WeisfeilerLehman over SubgraphMatching on the device (one clique enumeration for every WL level): == against the
real reference's goldens, and bit for bit against the per-level device route -- n_iter + 1 SubgraphMatching runs on
the level-labelled elements, summed and normalised on the host as the reference does -- at the benchmark's scale."""
import os
import sys

import numpy as np
import pytest

import wl_sm_cases as cases
import wl_sm_oracle as oracle
from grakel_b200 import Graph, GraphKernel, SubgraphMatching, WeisfeilerLehman, _lib
from grakel_b200.kernels import sm_level_features

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "wl_sm.npz"))
RUNS = [(name, n_iter) for name, (_, _, _, n_iters) in sorted(cases.cases().items()) for n_iter in n_iters]


def wl(params, n_iter, normalize=False):
    return WeisfeilerLehman(n_iter=n_iter, normalize=normalize, base_graph_kernel=(SubgraphMatching, dict(params)))


@pytest.mark.parametrize("name,n_iter", RUNS)
def test_goldens(name, n_iter):
    X, Y, params, _ = cases.cases()[name]
    if name in cases.GRAPH_OBJECT_CASES:
        X, Y = [Graph(*x) for x in X], [Graph(*y) for y in Y]
    for norm in (False, True):
        key = "%s_%d%s" % (name, n_iter, "_norm" if norm else "")
        k = wl(params, n_iter, norm)
        np.testing.assert_array_equal(k.fit_transform(X), G[key + "_fit_transform"])
        np.testing.assert_array_equal(k.diagonal(), G[key + "_ft_diag"])
        np.testing.assert_array_equal(k.transform(Y), G[key + "_ft_transform"])
        k = wl(params, n_iter, norm)
        np.testing.assert_array_equal(k.fit(X).transform(Y), G[key + "_fit_transform_y"])
        xd, yd = k.diagonal()
        np.testing.assert_array_equal(xd, G[key + "_fit_diag_x"])
        np.testing.assert_array_equal(yd, G[key + "_fit_diag_y"])


def per_level(params, n_iter, X, Y=None, normalize=False):
    """The per-level device route: one SubgraphMatching per WL level on the level's labels, K summed in level order;
    normalised by the sum's diagonal (fit_transform) or the level-ordered sums of the base diagonals (transform)."""
    Ks, dx, dy = [], [], []
    for lx, ly in oracle.level_elements(X, Y, n_iter):
        sm = SubgraphMatching(**params)
        if ly is None:
            Ks.append(sm.fit_transform(lx))
        else:
            Ks.append(sm.fit(lx).transform(ly))
            xd, yd = sm.diagonal()
            dx.append(xd)
            dy.append(yd)
    K = np.sum(Ks, axis=0)
    if not normalize:
        return K
    d = np.diagonal(K)
    outer = np.outer(d, d) if Y is None else np.outer(np.sum(dy, axis=0), np.sum(dx, axis=0))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.nan_to_num(np.divide(K, np.sqrt(outer)))


def bench_workload(n):
    from bench import gen_list
    return [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in gen_list(n, 40, 0)]


@pytest.mark.parametrize("k_sm", [3, 4])
def test_bench_scale_equals_the_per_level_route(k_sm):
    """bench.gen_list(2000, 40, 0) with edge labels (L_u + L_v) % 3, n_iter = 5: fit_transform and a 1500 / 500
    transform, normalize off and on."""
    X = bench_workload(2000)
    p = {"k": k_sm}
    K = per_level(p, 5, X)
    np.testing.assert_array_equal(wl(p, 5).fit_transform(X), K)
    with np.errstate(invalid="ignore", divide="ignore"):
        d = np.diagonal(K)
        Kn = np.nan_to_num(np.divide(K, np.sqrt(np.outer(d, d))))
    np.testing.assert_array_equal(wl(p, 5, True).fit_transform(X), Kn)
    Xf, Y = X[:1500], X[1500:]
    np.testing.assert_array_equal(wl(p, 5).fit(Xf).transform(Y), per_level(p, 5, Xf, Y))
    np.testing.assert_array_equal(wl(p, 5, True).fit(Xf).transform(Y), per_level(p, 5, Xf, Y, normalize=True))


def wl_counts(k, n_fit, rows):
    """gk_sm_wl_counts of `rows` for the estimator's fitted graphs (the setup of the SubgraphMatching level route)."""
    with _lib.engine() as eng:
        classes = k._level_classes(eng, k.X.block, k.X.ids)
        sm_level_features(eng, k._sm, k.X.base, classes, True, k._n_iter - 1)
        return [eng.sm_wl_counts(n_fit, r) for r in rows]


def level_counts(params, n_iter, X, rows):
    """gk_sm_counts of every level's SubgraphMatching, per row: [n, n_iter + 1, k + 1]."""
    out = [[] for _ in rows]
    for lx, _ in oracle.level_elements(X, None, n_iter):
        sm = SubgraphMatching(**params)
        sm.initialize()
        gp, rp, ci, ids, elids, vt, et, flags = sm._pack(sm.parse_input(lx))
        with _lib.engine() as eng:
            eng.pack(gp, rp, ci, ids, None, None)
            eng.sm_features(int(sm.k), sm.lambdas_, vt, et, elids, flags)
            for i, r in enumerate(rows):
                out[i].append(eng.sm_counts(len(X), r))
    return [np.stack(o, axis=1) for o in out]


def test_level_counts_equal_the_per_level_counts():
    X = bench_workload(2000)[:400]
    p = {"k": 4}
    k = wl(p, 5).fit(X)
    rows = [0, 17, 233, 399]
    for a, b in zip(wl_counts(k, len(X), rows), level_counts(p, 5, X, rows)):
        np.testing.assert_array_equal(a, b)
    Xs = cases.fit_set()
    k = wl({}, 2).fit(Xs)
    np.testing.assert_array_equal(wl_counts(k, len(Xs), [3])[0], oracle.level_counts({}, 2, Xs, 3))


@pytest.mark.parametrize("params", [{"k": 4}, {"k": 4, "ke": cases.ke_half}])
def test_level_route_row_ranges_and_device_output(params, monkeypatch):
    """Staged and global records give the same K (exact and real sums); so do row ranges and device output."""
    X = bench_workload(300)
    Xf, Y = X[:220], X[220:]
    k = wl(params, 3)
    K = k.fit_transform(Xf)
    Kt = k.transform(Y)
    Kr, _, _ = k._base_run(k.X, len(Xf), row_range=(7, 131))
    np.testing.assert_array_equal(Kr, K[7:131])
    import torch
    dev = torch.zeros((len(Xf), len(Xf)), dtype=torch.float64, device="cuda")
    k._base_run(k.X, len(Xf), device_ptr=dev.data_ptr())
    torch.cuda.synchronize()
    np.testing.assert_array_equal(dev.cpu().numpy(), K)
    monkeypatch.setenv("GRAKEL_B200_SM_GLOBAL", "1")
    np.testing.assert_array_equal(wl(params, 3).fit_transform(Xf), K)
    np.testing.assert_array_equal(wl(params, 3).fit(Xf).transform(Y), Kt)


def test_n_iter_cap():
    """(n_iter + 1) * min(k, largest graph) may be 64: k = 4 on graphs of 4 or more vertices allows n_iter = 15."""
    X = bench_workload(12)
    p = {"k": 4}
    np.testing.assert_array_equal(wl(p, 15).fit_transform(X), per_level(p, 15, X))
    with pytest.raises(NotImplementedError, match="more than 64"):
        wl(p, 16).fit_transform(X)


def test_dist_is_refused():
    X = cases.fit_set()
    k = wl({}, 2).fit(X)
    sm, data = k._sm, k.X.base
    gp, rp, ci, _, elids, _, et, flags = sm._pack(data.graphs)
    with _lib.engine() as eng:
        eng.pack(gp, rp, ci, None, None, None)
        eng.sm_wl_features(5, 2, None, sm.lambdas_, et, elids, _lib.GK_SM_KV_NONE | (flags & ~3))
        with pytest.raises(NotImplementedError, match="GK_DIST"):
            eng.gram(len(X), dist=True)


def test_graph_kernel_dispatch():
    X, Y = cases.fit_set(), cases.transform_set()
    K = wl({"k": 3}, 2).fit_transform(X)
    for spec in ([{"name": "WL", "n_iter": 2}, {"name": "SM", "k": 3}],
                 [{"name": "weisfeiler_lehman", "n_iter": 2}, {"name": "subgraph_matching", "k": 3}]):
        np.testing.assert_array_equal(GraphKernel(kernel=spec).fit_transform(X), K)
    np.testing.assert_array_equal(GraphKernel(kernel=["WL", "SM"]).fit_transform(X), wl({}, 5).fit_transform(X))
