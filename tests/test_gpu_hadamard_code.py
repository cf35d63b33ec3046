"""HadamardCode on the device: every golden K of the reference bit for bit (normalised ones included), the level vectors
of gk_hc_vectors against the reference's tuples (the wrapped case included), the width-growth transform, the
ShortestPath base in both path-sum orders, the EdgeHistogram base, GraphKernel, the collision retry, and the full-size
benchmark workload against the NumPy restatement with row blocks, pitched and device output."""
import os
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import hc_oracle  # noqa: E402
from grakel_b200 import EdgeHistogram, GraphKernel, HadamardCode, ShortestPath, _lib, kernels  # noqa: E402
from test_hadamard_code import CASES, GOLDEN, INPUTS  # noqa: E402
from make_golden_hadamard_code import GK_FORMS, same_width  # noqa: E402

pytestmark = pytest.mark.gpu


def _est(spec):
    base = spec.get("base", "VH")
    bk = None if base == "VH" else EdgeHistogram if base == "EH" else (ShortestPath, dict(base[1]))
    return HadamardCode(n_iter=spec["n_iter"], base_graph_kernel=bk, normalize=spec.get("normalize", False),
                        n_jobs=spec.get("n_jobs"))


def _same(a, b):
    a = np.asarray(a)
    assert a.shape == b.shape and np.array_equal(a, b), (a - b)[np.nonzero(a != b)][:5] if a.shape == b.shape else a.shape


@pytest.mark.parametrize("name,spec", CASES, ids=lambda x: str(x))
def test_golden_cases(name, spec):
    hc = _est(spec)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        K = hc.fit_transform(spec["X"])
        _same(K, GOLDEN[name + "__K"])
        if spec.get("Y") is not None:
            _same(hc.transform(spec["Y"]), GOLDEN[name + "__Kt"])
            if spec.get("normalize"):
                xd, yd = hc.diagonal()
                _same(np.asarray(xd).ravel(), GOLDEN[name + "__xd"])
                _same(np.asarray(yd).ravel(), GOLDEN[name + "__yd"])


@pytest.mark.parametrize("name,spec", [c for c in CASES if c[1].get("vec")], ids=lambda x: str(x))
def test_level_vectors(name, spec):
    hc = HadamardCode(n_iter=spec["n_iter"]).fit(spec["X"])
    for lv in range(spec["n_iter"]):
        _same(hc.hc_vectors(spec["X"], lv), GOLDEN["%s__vec%d" % (name, lv)])


def test_width_growth_transform():
    """gen8: the transform labels push nl from 4 to 5 labels, W from 4 to 8: K is zero, Y_diag is each Y graph's own
    self similarity at the new width, X_diag the fitted one."""
    spec = INPUTS["gen8_vh"]
    hc = HadamardCode(n_iter=3).fit(spec["X"])
    assert hc._width == 4
    K = hc.transform(spec["Y"])
    assert K.shape == (len(spec["Y"]), len(spec["X"])) and not K.any()
    xd, yd = hc.diagonal()
    Ky, _ = hc_oracle.kernel(spec["Y"], 3)
    Kx, _ = hc_oracle.kernel(spec["X"], 3)
    _same(np.asarray(yd), np.diag(Ky))
    _same(np.asarray(xd), np.diag(Kx))


@pytest.mark.parametrize("name", ["sp_fw", "sp_dj"])
def test_sp_path_sum_orders(name):
    spec = INPUTS[name]
    hc = _est(spec)
    hc.fit(spec["X"])
    assert hc._dijkstra_order(hc.X.block) == (name == "sp_dj")
    _same(hc.fit_transform(spec["X"]), GOLDEN[name + "__K"])


def test_eh_is_n_iter_times_edge_histogram():
    spec = INPUTS["eh"]
    K = _est(spec).fit_transform(spec["X"])
    _same(K, spec["n_iter"] * EdgeHistogram().fit_transform(spec["X"]))


@pytest.mark.parametrize("name", sorted(GK_FORMS))
def test_graph_kernel_forms(name):
    _same(GraphKernel(kernel=GK_FORMS[name]).fit_transform(same_width()), GOLDEN[name + "__K"])


def test_collision_retry():
    """A degenerate first hash (every z_c = 0) puts every vertex in one slot; the verification must see it, and the
    retry with a fresh seed must give the reference's classes."""
    spec = INPUTS["directed"]
    hc = HadamardCode(n_iter=spec["n_iter"]).fit(spec["X"])
    block = hc.X.block
    with _lib.engine() as eng:
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, hc.X.ids)
        eng.selftest_hc_collision()
        st = eng.hc_features(spec["n_iter"], hc._width, skip=hc.X.skip)
        assert st.hash_retries >= 1
        K, _, _ = eng.gram(block.n_graphs)
        st2 = eng.hc_features(spec["n_iter"], hc._width, skip=hc.X.skip)
        assert st2.hash_retries == 0
    _same(K, GOLDEN["directed__K"])


def test_arguments_refused():
    spec = INPUTS["directed"]
    hc = HadamardCode(n_iter=2).fit(spec["X"])
    block = hc.X.block
    with _lib.engine() as eng:
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, hc.X.ids)
        for n_iter, width in ((2, 3), (0, 8), (64, 8), (2, 4)):  # not a power of two, n_iter range, label >= width
            with pytest.raises(_lib.GrakelB200Error):
                eng.hc_features(n_iter, width)


@pytest.fixture(scope="module")
def full():
    import bench
    X = bench.gen_list(10000, 40, 0)
    hc = HadamardCode(n_iter=5)
    K = hc.fit_transform(X)
    return X, hc, K


def test_full_size_symmetric_and_rows(full):
    X, hc, K = full
    assert K.shape == (10000, 10000) and np.array_equal(K, K.T)
    rows = np.random.RandomState(0).choice(len(X), 6, replace=False)
    sub = [X[i] for i in rows]
    # the restatement over the sampled graphs and a seeded column sample (the enumeration of all graphs is 0..6)
    cols = np.random.RandomState(1).choice(len(X), 200, replace=False)
    Ko, _ = hc_oracle.kernel([X[i] for i in cols], 5, sub)
    assert hc._width == kernels.hc_width(len(hc_oracle.enumerate_labels(x[1] for x in [X[i] for i in cols] + sub))) == 8
    _same(K[np.ix_(rows, cols)], Ko)


def test_full_size_diagonal_and_outputs(full):
    X, hc, K = full
    _same(np.asarray(hc._X_diag), np.diag(K).copy())
    data = hc.X
    block = data.block
    with _lib.engine() as eng:
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, data.ids)
        eng.hc_features(5, hc._width, skip=data.skip)
        Kr, _, _ = eng.gram(block.n_graphs, row_range=(1000, 3517))
        _same(Kr, K[1000:3517])
        import torch  # pitched device output
        ld = block.n_graphs + 40
        d = torch.full((block.n_graphs, ld), -1.0, dtype=torch.float64, device="cuda:%d" % eng.device)
        eng.gram(block.n_graphs, device_ptr=d.data_ptr(), ld=ld)
        torch.cuda.synchronize()
        _same(d[:, :block.n_graphs].cpu().numpy(), K)
