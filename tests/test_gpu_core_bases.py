"""CoreFramework over NeighborhoodHash, OddSth, WeisfeilerLehmanOptimalAssignment and SubgraphMatching on the device:
K and the diagonals of every golden of tests/golden/core_bases.npz (the real reference's) with ==, the reference's
errors, the bench graphs against the per-level base kernels folded on the host, and the fold's level order check."""
import os
import sys
import warnings

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import core_bases_cases as cases  # noqa: E402

from grakel_b200 import (CoreFramework, GraphKernel, NeighborhoodHash, OddSth, SubgraphMatching,  # noqa: E402
                         WeisfeilerLehmanOptimalAssignment, _lib)

pytestmark = pytest.mark.gpu

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "core_bases.npz"))
KINDS = {"NH": NeighborhoodHash, "ODD": OddSth, "WLOA": WeisfeilerLehmanOptimalAssignment, "SM": SubgraphMatching}
OPEN = [n for n, (kind, p) in cases.BASES.items() if kind != "SM" or p.get("ke", "x") is None]


def core(name, normalize):
    np.random.seed(cases.GLOBAL_SEED)  # the "nhgl" case draws from numpy's global stream, as its golden did
    kind, params = cases.params_of(name)
    return CoreFramework(normalize=normalize, base_graph_kernel=(KINDS[kind], params))


def check(key, fn):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if key + "_error" in GOLD:
            etype, msg = GOLD[key + "_error"]
            with pytest.raises(Exception) as ei:
                fn()
            assert type(ei.value).__name__ == etype and str(ei.value) == msg
            return
        res = fn()
    if isinstance(res, tuple):
        for i, r in enumerate(res):
            assert np.array_equal(np.asarray(r, dtype=np.float64), GOLD["%s_%d" % (key, i)]), (key, i)
    else:
        assert np.array_equal(np.asarray(res, dtype=np.float64), GOLD[key]), key


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("name", OPEN)
def test_core_bases_golden(name, norm):
    tag = name + ("_norm" if norm else "")
    X, Y, Z, U = cases.fit_set(), cases.transform_set(), cases.isolated_set(), cases.unlabelled_edges_set()
    for key, data in (("_fit_transform", X), ("_isolated", Z)):
        k = core(name, norm)
        check(tag + key, lambda: k.fit_transform(data))
    k = core(name, norm)
    check(tag + "_ft_transform", lambda: (k.fit_transform(X), k.transform(Y))[1])
    check(tag + "_ft_transform_diag", k.diagonal)
    k = core(name, norm)
    check(tag + "_fit_transform_y", lambda: k.fit(X).transform(Y))
    check(tag + "_fit_transform_y_diag", k.diagonal)
    k = core(name, norm)
    check(tag + "_isolated_fit", lambda: k.fit(Z).transform(X))
    k = core(name, norm)
    check(tag + "_unlabelled_edges_fit", lambda: k.fit(U).transform(Y))


def test_core_sm_with_edge_kernel_refused():
    with pytest.raises(NotImplementedError):
        CoreFramework(base_graph_kernel=SubgraphMatching).fit_transform(cases.fit_set())


def host_fold(name, X, Y=None):
    """The reference's per-level fold (core_framework.py:177-223) over this package's base kernels, each level's K
    fetched to the host and scattered there."""
    from grakel_b200.core_framework import core_numbers, level_blocks
    from grakel_b200.packing import pack
    kind, params = cases.BASES[name]

    def levels(D):
        b = pack(D, "sp", need_labels=True, len_ok=lambda n: n >= 1, want_weights=True)
        return b.n_graphs, {lv: (idx, lb) for lv, idx, lb in level_blocks(b, core_numbers(b))}
    nx, fl = levels(X)
    fitted, K = {}, np.zeros((nx, nx))
    for lv in sorted(fl, reverse=True):
        idx, els = fl[lv]
        fitted[lv] = KINDS[kind](**params)
        Ki = fitted[lv].fit_transform(els)
        for j in range(len(idx)):
            K[idx[j], idx] += Ki[j, :]
    if Y is None:
        return K
    ny, tl = levels(Y)
    Kt = np.zeros((ny, nx))
    for lv in sorted(tl, reverse=True):
        if lv not in fl or not len(tl[lv][0]):
            continue
        idx, els = tl[lv]
        Ki = fitted[lv].transform(els)
        for j in range(len(idx)):
            Kt[idx[j], fl[lv][0]] += Ki[j, :]
    return Kt


@pytest.mark.parametrize("name", ["nh", "nhcs", "oddN", "odd2", "wloa", "smN"])
def test_core_bases_bench_graphs(name):
    import bench
    G = bench.gen_list(2000, 40, 0)
    if name == "smN":  # the reference's SubgraphMatching reads edge labels even with ke=None
        G = [[g, L, {e: 1 for e in g}] for g, L in G]
    X, Y = G[:1500], G[1500:]
    k = core(name, False)
    K = k.fit_transform(X)
    assert set(k.stage_times_) == {"levels", "base", "fold"}
    assert np.array_equal(K, host_fold(name, X))
    assert np.array_equal(k.transform(Y), host_fold(name, X, Y))


def test_core_fold_level_order():
    """Levels must be added in strictly descending core order; a refused call leaves the sum as it was."""
    k = NeighborhoodHash(random_state=0)
    X = cases.fit_set()
    k.fit(X)
    b = k.X.block
    eng = _lib.get_engine()
    eng.core_sum_begin(b.n_graphs, b.n_graphs, True)
    rows = np.arange(b.n_graphs)

    def level(lv):
        eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, k.X.ids, None, None)
        eng.nh_features(k.R, k._nh_code, k.bits, k.X.codes, k.X.valid)
        eng.core_level_add(lv, b.n_graphs, rows, rows, b.n_graphs, want_diag=False)
    level(2)
    with pytest.raises(_lib.GrakelB200Error):
        level(3)
    with pytest.raises(_lib.GrakelB200Error):
        level(2)
    with pytest.raises(_lib.GrakelB200Error):  # a repeated row
        eng.core_level_add(1, b.n_graphs, np.zeros(b.n_graphs), rows, b.n_graphs, want_diag=False)
    level(0)
    K, _ = eng.wl_level_sum_fetch(b.n_graphs, b.n_graphs)
    Kn = k._nh_run(b, k.X.ids, k.X.codes, k.X.valid, b.n_graphs)
    assert np.array_equal(K, Kn + Kn)


@pytest.mark.parametrize("base", ["NH", "ODD", "WL-OA", "SM"])
def test_core_bases_dispatch(base):
    X = [[g, L, E] for g, L, E in cases.fit_set()]
    params = {"NH": {"random_state": 0}, "SM": {"k": 3, "ke": None}}.get(base, {})
    K = GraphKernel(kernel=["CORE", dict(name=base, **params)]).fit_transform(X)
    cls = {"NH": NeighborhoodHash, "ODD": OddSth, "WL-OA": WeisfeilerLehmanOptimalAssignment, "SM": SubgraphMatching}
    ref = CoreFramework(base_graph_kernel=(cls[base], params)).fit_transform(X)
    assert np.array_equal(K, ref)
