"""GraphletSampling on the device: K, the diagonals and the MT19937 state equal the reference's goldens with ==, the
(graph, class) count tables equal the oracle's, and what the device refuses is refused before any draw."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
import gs_cases  # noqa: E402
import gs_oracle  # noqa: E402
from grakel_b200 import Graph, GraphletSampling, _lib  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(gs_cases.GOLDEN)
UNDIRECTED = [c for c in gs_cases.CASES if not gs_cases.directed(c[1])]
DIRECTED = [c for c in gs_cases.CASES if gs_cases.directed(c[1])]


def _graphs(key):
    sizes, flat = G[key + "_sizes"], G[key + "_adj"]
    out, o = [], 0
    for n in sizes:
        out.append(flat[o:o + n * n].reshape(n, n))
        o += n * n
    return out


@pytest.mark.parametrize("case", UNDIRECTED, ids=[c[0] for c in UNDIRECTED])
@pytest.mark.parametrize("norm", [False, True])
def test_golden(case, norm):
    name, _, k, sampling, form, seed = case
    X = [gs_cases.element(A, form, Graph) for A in _graphs(name + "_X")]
    Y = [gs_cases.element(A, form, Graph) for A in _graphs(name + "_Y")]
    tag = "%s_n%d" % (name, norm)
    gk = GraphletSampling(k=k, sampling=dict(sampling), random_state=seed, normalize=norm)
    with np.errstate(all="ignore"):
        Kf = gk.fit_transform(X)
        st = gk.random_state_.get_state()
        assert np.array_equal(st[1], G[tag + "_mt_fit"]) and st[2] == G[tag + "_pos_fit"]
        Kt = gk.transform(Y)
    np.testing.assert_array_equal(Kf, G[tag + "_Kf"])
    np.testing.assert_array_equal(Kt, G[tag + "_Kt"])
    xd, yd = gk.diagonal()
    np.testing.assert_array_equal(xd, G[tag + "_xdiag"])
    np.testing.assert_array_equal(yd, G[tag + "_ydiag"])
    st = gk.random_state_.get_state()
    assert np.array_equal(st[1], G[tag + "_mt"]) and st[2] == G[tag + "_pos"]


@pytest.mark.parametrize("case", DIRECTED, ids=[c[0] for c in DIRECTED])
def test_directed_refused_before_draws(case):
    name, _, k, sampling, form, seed = case
    X = [gs_cases.element(A, form, Graph) for A in _graphs(name + "_X")]
    gk = GraphletSampling(k=k, sampling=dict(sampling), random_state=seed)
    with pytest.raises(NotImplementedError, match="non-symmetric"):
        gk.fit_transform(X)
    assert gk.random_state_.get_state()[2] == np.random.RandomState(seed).get_state()[2]


@pytest.mark.parametrize("k", [3, 4, 5, 6])
def test_count_tables_equal_oracle(k):
    """Every graph's (class, samples, count) rows on 500 random graphs of 3 .. 40 vertices, loops included, against
    the oracle's classes and counts, fit and transform."""
    rs = np.random.RandomState(100 + k)
    mats = [gs_cases.rand_adj(rs, n, p, loops=0.1) for n, p in zip(rs.randint(3, 41, size=500), rs.uniform(0.05, 0.5, 500))]
    X, Y = mats[:400], mats[400:]
    n = 40 if k < 6 else 15
    gk = GraphletSampling(k=k, sampling={"n_samples": n}, random_state=k)
    Kf = gk.fit_transform([[A] for A in X])
    Kt = gk.transform([[A] for A in Y])
    ors = np.random.RandomState(k)
    cx = gs_oracle.counts([gs_oracle.graph_classes(A, k, n, ors) for A in X])
    cy = gs_oracle.counts([gs_oracle.graph_classes(A, k, n, ors) for A in Y], set().union(*cx))
    base = [sum(1 << (j * (j - 1) // 2 + j) for j in range(m)) for m in range(8)]
    for rows, want, g0 in ((gk.X, cx, 0), (gk.Y_, cy, len(X))):
        got = [dict() for _ in want]
        for g, code, samples, count in rows:
            got[g - g0][int(code)] = int(count)
        assert got == [{base[m] + p: v for (m, p), v in c.items()} for c in want]
    np.testing.assert_array_equal(Kf, gs_oracle.gram(cx, cx))
    np.testing.assert_array_equal(Kt, gs_oracle.gram(cy, cx))


BASE = [sum(1 << (j * (j - 1) // 2 + j) for j in range(m)) for m in range(8)]


def _as_rows(cl):
    return [{BASE[m] + p: v for (m, p), v in c.items()} for c in cl]


def _table(rows, n, g0):
    got = [dict() for _ in range(n)]
    for g, code, samples, count in rows:
        got[g - g0][int(code)] = int(count)
    return got


@pytest.mark.parametrize("k", [3, 4, 5, 6])
def test_bench_graphs_default_bound_equal_oracle(k):
    """bench.gen_list(500, 40, 0) at the default bound {"epsilon": 0.05} (2 005 .. 13 805 samples per graph), fit on
    400 graphs and transform of the other 100 plus four graphs of 150 .. 300 vertices: every graph's count table and
    K against the oracle's classes of the same draws (the draws themselves equal numpy's: test_graphlet_sampling)."""
    X = [el[0] for el in bench.gen_list(500, 40, 0, as_adj=True)]
    rs = np.random.RandomState(k)
    X += [gs_cases.rand_adj(rs, n, 4.0 / n) for n in (150, 200, 257, 300)]
    fit, new = X[:400], X[400:]
    gk = GraphletSampling(k=k, sampling={"epsilon": 0.05}, random_state=k)
    Kf = gk.fit_transform([[A] for A in fit])
    Kt = gk.transform([[A] for A in new])
    n = gs_oracle.n_samples_of({"epsilon": 0.05}, k)
    ors = np.random.RandomState(k)
    cls = []
    for part in (fit, new):
        size, idx = _lib.gs_draw(ors, [A.shape[0] for A in part], k, n)
        io = 0
        for g, A in enumerate(part):
            sz = size[g * n:(g + 1) * n]
            cls.append(gs_oracle.classes_of_draws(A, sz, idx[io:io + int(sz.sum())]))
            io += int(sz.sum())
    cx = gs_oracle.counts(cls[:400])
    cy = gs_oracle.counts(cls[400:], set().union(*cx))
    assert _table(gk.X, len(fit), 0) == _as_rows(cx)
    assert _table(gk.Y_, len(new), len(fit)) == _as_rows(cy)
    np.testing.assert_array_equal(Kf, gs_oracle.gram(cx, cx))
    np.testing.assert_array_equal(Kt, gs_oracle.gram(cy, cx))


def test_read_tu_block(tmp_path):
    """A datasets.read_tu block gives the K of the same graphs as edge dictionaries (rows in sorted vertex order)."""
    from tu_io import write_tu
    from grakel_b200.datasets import read_tu
    rs = np.random.RandomState(0)
    els, dicts, base = [], [], 1
    for n in rs.randint(5, 30, size=40):
        E = {(i, (i + 1) % n) for i in range(n)} | {tuple(int(x) for x in rs.choice(n, 2, replace=False))
                                                    for _ in range(n // 2)}
        E |= {(b, a) for a, b in E}
        els.append([[(a + base, b + base) for a, b in sorted(E)], {v + base: 1 for v in range(n)}])
        dicts.append([{u + base: {v + base: 1.0 for a, v in E if a == u} for u in range(n)}])
        base += n
    write_tu(str(tmp_path), "GS", els, classes=[0] * len(els))
    block = read_tu(str(tmp_path), "GS", kernel="SP").data
    assert block.n_graphs == 40
    a = GraphletSampling(k=4, sampling={"n_samples": 200}, random_state=3, normalize=True)
    b = GraphletSampling(k=4, sampling={"n_samples": 200}, random_state=3, normalize=True)
    np.testing.assert_array_equal(a.fit_transform(block), b.fit_transform(dicts))
    assert np.array_equal(a.X, b.X)


def test_row_range_and_device_output():
    import torch
    name, _, k, sampling, form, seed = UNDIRECTED[0]
    X = _graphs(name + "_X")
    gk = GraphletSampling(k=k, sampling=dict(sampling), random_state=seed)
    gk.initialize()
    els = gk._elements([[A] for A in X])
    out = torch.zeros((3, len(X)), dtype=torch.float64, device="cuda")
    gk._gs_run(els, want_matrix=False, device_ptr=out.data_ptr(), row_range=(2, 5))
    np.testing.assert_array_equal(out.cpu().numpy(), G[name + "_n0_Kf"][2:5])


def test_limits_and_bad_indexes_raise():
    X = [[np.ones((4, 4)) - np.eye(4)]]
    gk = GraphletSampling(k=7, sampling={"n_samples": 3}, random_state=1)
    with pytest.raises(NotImplementedError, match="more than 6"):
        gk.fit_transform(X)
    assert gk.random_state_.get_state()[2] == np.random.RandomState(1).get_state()[2]
    with _lib.engine(None) as eng:
        eng.pack([0, 4], [0, 3, 6, 9, 12], [1, 2, 3, 0, 2, 3, 0, 1, 3, 0, 1, 2])
        # argument checks, before any launch
        with pytest.raises(_lib.GrakelB200Error, match="larger than k"):
            eng.gs_features(3, 1, 0, [0, 1], np.array([4], np.uint8), np.array([0, 1, 2, 3], np.int32))
        with pytest.raises(_lib.GrakelB200Error, match="does not match the sizes"):
            eng.gs_features(5, 1, 0, [0, 1], np.array([3], np.uint8), np.array([0, 1], np.int32))
        # an index outside its graph: found by the classification kernel, no feature block left for gk_gram
        with pytest.raises(_lib.GrakelB200Error, match="not a vertex"):
            eng.gs_features(5, 1, 0, [0, 1], np.array([3], np.uint8), np.array([0, 1, 4], np.int32))
        with pytest.raises(_lib.GrakelB200Error, match="no feature block"):
            eng.gram(1)
        # fp64 only: an fp32 K could not hold entries above 2^24 exactly
        eng.gs_features(5, 1, 0, [0, 1], np.array([3], np.uint8), np.array([0, 1, 3], np.int32))
        with pytest.raises(NotImplementedError, match="fp64 only"):
            eng.gram(1, dtype=np.float32)
