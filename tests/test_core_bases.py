"""CoreFramework over NeighborhoodHash, OddSth, WeisfeilerLehmanOptimalAssignment and SubgraphMatching, host side:
the level blocks in the reference's get_subgraph shape, a host restatement of the per-level fold over OddSth against
the reference's goldens, the dispatch, and the bases that stay refused before any device work."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import core_bases_cases as cases  # noqa: E402
import odd_oracle  # noqa: E402

from grakel_b200 import (CoreFramework, GraphHopper, GraphKernel, GraphletSampling, HadamardCode,
                         MultiscaleLaplacian, NeighborhoodSubgraphPairwiseDistance, Propagation, PyramidMatch,
                         RandomWalk, ShortestPathAttr, SubgraphMatching, SvmTheta, EdgeHistogram, OddSth)
from grakel_b200.core_framework import core_numbers, level_blocks
from grakel_b200.kernels import odd_label_tables
from grakel_b200.packing import Graph, pack

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "core_bases.npz"))

TRIANGLE_TAIL = {(0, 1): 1, (1, 0): 1, (1, 2): 1, (2, 1): 1, (0, 2): 1, (2, 0): 1, (2, 3): 1, (3, 2): 1}


def levels(X):
    b = pack(X, "sp", need_labels=True, len_ok=lambda n: n >= 1, want_weights=True)
    return level_blocks(b, core_numbers(b))


def rows_of(lb, k):
    a, z = int(lb.graph_ptr[k]), int(lb.graph_ptr[k + 1])
    return {u - a: [int(w) - a for w in lb.col_idx[lb.row_ptr[u]:lb.row_ptr[u + 1]]] for u in range(a, z)}


@pytest.mark.parametrize("spelling", ["dict", "adjacency", "graph"])
def test_level_blocks_order(spelling):
    L = {0: "a", 1: "b", 2: "c", 3: "d"}
    g = TRIANGLE_TAIL
    if spelling == "adjacency":
        A = np.zeros((4, 4))
        for (u, v) in g:
            A[u, v] = 1
        g = A
    el = [g, L] if spelling != "graph" else Graph(g, L, {})
    out = levels([el, [{(0, 1): 1, (1, 0): 1}, {0: "a", 1: "a"}]])
    assert [lv for lv, *_ in out] == [2, 1, 0]
    lv2, idx2, b2 = out[0]
    assert idx2.tolist() == [0]
    assert rows_of(b2, 0) == {0: [1, 2], 1: [0, 2], 2: [0, 1]}
    assert b2.labels == ["a", "b", "c"] and b2.mode == "core"
    _, idx0, b0 = out[2]
    assert idx0.tolist() == [0, 1]
    assert rows_of(b0, 0) == {0: [1, 2], 1: [0, 2], 2: [0, 1, 3], 3: [2]} and rows_of(b0, 1) == {0: [1], 1: [0]}

@pytest.mark.parametrize("base", [PyramidMatch, Propagation, GraphletSampling, SvmTheta, MultiscaleLaplacian,
                                  ShortestPathAttr, GraphHopper, RandomWalk, HadamardCode, EdgeHistogram,
                                  NeighborhoodSubgraphPairwiseDistance])
def test_out_of_scope_bases_refused(base):
    with pytest.raises(NotImplementedError):
        CoreFramework(base_graph_kernel=base).fit_transform([[TRIANGLE_TAIL, {0: 1, 1: 1, 2: 1, 3: 1}]])


def test_sm_with_edge_kernel_refused():
    with pytest.raises(NotImplementedError):
        CoreFramework(base_graph_kernel=(SubgraphMatching, {"k": 3})).initialize()
    CoreFramework(base_graph_kernel=(SubgraphMatching, {"k": 3, "ke": None})).initialize()


@pytest.mark.parametrize("base,cls", [("NH", "NeighborhoodHash"), ("ODD", "OddSth"),
                                      ("WL-OA", "WeisfeilerLehmanOptimalAssignment"), ("SM", "SubgraphMatching")])
def test_dispatch_opens(base, cls):
    gk = GraphKernel(kernel=["CORE", {"name": base, "ke": None} if base == "SM" else base])
    gk.initialize()
    gk.kernel_.initialize()
    assert type(gk.kernel_) is CoreFramework and gk.kernel_.base_graph_kernel_.__name__ == cls and gk.kernel_._fold


def test_max_core_error():
    cf = CoreFramework(base_graph_kernel=OddSth)
    cf.min_core = 5  # the reference stores -1 at construction; a later assignment is validated at fit
    with pytest.raises(ValueError, match="The maximum core equals the min_core boundary set in init."):
        cf.fit(cases.fit_set())


def odd_level_gram(lx, ly, h):
    """OddSth's K of level blocks on the host (odd_oracle's DAG identities)."""
    def feats(b):
        ids, rank, strings = odd_label_tables(b.labels, b.graph_ptr)
        out = []
        for k in range(b.n_graphs):
            a, z = int(b.graph_ptr[k]), int(b.graph_ptr[k + 1])
            r = rows_of(b, k)
            out.append(odd_oracle.graph_features(z - a, [r[u] for u in range(z - a)], [strings[i] for i in ids[a:z]],
                                                 rank[a:z].tolist(), h))
        return out
    return odd_oracle.gram(feats(lx), None if ly is None else feats(ly))


def odd_fold(X, Y=None, h=None):
    """core_framework.py:177-223 restated: K[idx_j, idx] += K_i[j, :] from the largest core down, a transform adding
    only the levels the fit has."""
    fx = {lv: (idx, b) for lv, idx, b in levels(X)}
    nx = len(X)
    if Y is None:
        K = np.zeros((nx, nx))
        for lv in sorted(fx, reverse=True):
            idx, b = fx[lv]
            Ki = odd_level_gram(b, None, h)
            for j in range(len(idx)):
                K[idx[j], idx] += Ki[j, :]
        return K
    K = np.zeros((len(Y), nx))
    for lv, idx, b in levels(Y):
        if lv in fx and len(idx):
            Ki = odd_level_gram(fx[lv][1], b, h)
            for j in range(len(idx)):
                K[idx[j], fx[lv][0]] += Ki[j, :]
    return K


@pytest.mark.parametrize("name,h", [("oddN", None), ("odd2", 2)])
def test_fold_restatement_matches_reference(name, h):
    X, Y, Z, U = cases.fit_set(), cases.transform_set(), cases.isolated_set(), cases.unlabelled_edges_set()
    assert np.array_equal(odd_fold(X, h=h), GOLD[name + "_fit_transform"])
    assert np.array_equal(odd_fold(Z, h=h), GOLD[name + "_isolated"])
    assert np.array_equal(odd_fold(X, Y, h=h), GOLD[name + "_ft_transform"])
    assert np.array_equal(odd_fold(X, Y, h=h), GOLD[name + "_fit_transform_y"])
    assert np.array_equal(odd_fold(Z, X, h=h), GOLD[name + "_isolated_fit"])
    assert np.array_equal(odd_fold(U, Y, h=h), GOLD[name + "_unlabelled_edges_fit"])
    K = odd_fold(X, h=h)
    d = np.diagonal(K)
    with np.errstate(divide="ignore", invalid="ignore"):
        assert np.array_equal(np.nan_to_num(K / np.sqrt(np.outer(d, d))), GOLD[name + "_norm_fit_transform"])


def test_sm_missing_edge_labels_raise_at_fit():
    """The reference's SubgraphMatching reads every level subgraph's edge labels, even with ke=None."""
    for data in (cases.isolated_set(), cases.unlabelled_edges_set()):
        cf = CoreFramework(base_graph_kernel=(SubgraphMatching, {"k": 3, "ke": None}))
        with pytest.raises(ValueError, match="Graph does not have any labels for edges."):
            cf.fit(data)


def test_fold_flag_missing_on_old_estimators():
    cf = CoreFramework(base_graph_kernel=OddSth)
    cf.initialize()
    del cf._fold  # as on an estimator pickled before the fold route existed
    with pytest.raises(Exception) as e:
        cf.diagonal()
    assert not isinstance(e.value, AttributeError) or "_fold" not in str(e.value)

