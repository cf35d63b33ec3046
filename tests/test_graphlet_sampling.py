"""GraphletSampling on the host: the oracle against the reference's goldens, the library's MT19937 draws against
numpy and the goldens, the reference's errors and warnings, and GraphKernel's dispatch."""
import os
import sys
import warnings

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gs_cases  # noqa: E402
import gs_oracle  # noqa: E402
from grakel_b200 import GraphKernel, GraphletSampling, _lib  # noqa: E402

G = np.load(gs_cases.GOLDEN)


def _graphs(key):
    sizes, flat = G[key + "_sizes"], G[key + "_adj"]
    out, o = [], 0
    for n in sizes:
        out.append(flat[o:o + n * n].reshape(n, n))
        o += n * n
    return out


@pytest.mark.parametrize("case", gs_cases.CASES, ids=[c[0] for c in gs_cases.CASES])
@pytest.mark.parametrize("norm", [False, True])
def test_oracle_equals_reference(case, norm):
    name, gname, k, sampling, _, seed = case
    if gs_cases.directed(gname):
        pytest.skip("directed samples are classified by bliss's canonical labeling, which the oracle does not restate")
    if k == 6 and norm:
        pytest.skip("the k = 6 oracle is slow; normalize off covers its counts")
    X, Y = _graphs(name + "_X"), _graphs(name + "_Y")
    rs = np.random.RandomState(seed)
    Kf, cx = gs_oracle.fit_transform(X, k, sampling, rs, normalize=norm)
    tag = "%s_n%d" % (name, norm)
    assert np.array_equal(rs.get_state()[1], G[tag + "_mt_fit"]) and rs.get_state()[2] == G[tag + "_pos_fit"]
    Kt, _ = gs_oracle.transform(Y, cx, k, sampling, rs, normalize=norm)
    np.testing.assert_array_equal(Kf, G[tag + "_Kf"])
    np.testing.assert_array_equal(Kt, G[tag + "_Kt"])
    assert np.array_equal(rs.get_state()[1], G[tag + "_mt"]) and rs.get_state()[2] == G[tag + "_pos"]


@pytest.mark.parametrize("case", gs_cases.CASES, ids=[c[0] for c in gs_cases.CASES])
def test_library_draws_equal_reference(case):
    """gk_gs_draw's sizes and index arrays are the ones the reference's `choice` returned, in order."""
    name, _, k, sampling, _, seed = case
    X, Y = _graphs(name + "_X"), _graphs(name + "_Y")
    n = gs_oracle.n_samples_of(sampling, k)
    rs = np.random.RandomState(seed)
    sx, ix = _lib.gs_draw(rs, [A.shape[0] for A in X], k, n)
    sy, iy = _lib.gs_draw(rs, [A.shape[0] for A in Y], k, n)
    np.testing.assert_array_equal(np.concatenate([sx, sy]), G[name + "_drawn_sizes"])
    np.testing.assert_array_equal(np.concatenate([ix, iy]), G[name + "_drawn"])
    assert np.array_equal(rs.get_state()[1], G[name + "_n0_mt"]) and rs.get_state()[2] == G[name + "_n0_pos"]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 7, 129, 300])
def test_library_draws_equal_numpy_above_128(n):
    rs, ref = np.random.RandomState(n), np.random.RandomState(n)
    size, idx = _lib.gs_draw(rs, [n], 5, 25)
    o = 0
    for t in range(25):
        lo, hi = min(3, n), min(5, n)
        r = lo if lo == hi else ref.randint(lo, hi + 1)
        assert size[t] == r
        np.testing.assert_array_equal(idx[o:o + r], ref.choice(list(range(n)), r, replace=False))
        o += r
    assert rs.randint(1 << 30) == ref.randint(1 << 30)


@pytest.mark.parametrize("name,params", gs_cases.ERROR_CASES, ids=[e[0] for e in gs_cases.ERROR_CASES])
def test_errors_match_reference(name, params):
    etype, msg = G["err_" + name]
    X = [[A] for A in _graphs("small_k3_X")]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception) as e:
            GraphletSampling(**params).fit(X)
    assert type(e.value).__name__ == etype and str(e.value) == msg


def test_warnings_and_limits_before_work():
    X = [[np.ones((3, 3))]]
    with pytest.warns(UserWarning, match="no implemented parallelization for GraphletSampling"):
        with pytest.raises(NotImplementedError):
            GraphletSampling(n_jobs=2).fit(X)
    with pytest.warns(UserWarning, match="graphlets are too big"):
        with pytest.raises(NotImplementedError, match="more than 6"):
            GraphletSampling(k=11, sampling={"n_samples": 2}).fit(X)
    with pytest.raises(NotImplementedError, match="more than 6"):
        GraphletSampling(k=7, sampling={"n_samples": 2}).fit(X)
    with pytest.raises(NotImplementedError, match="sampling=None"):
        GraphletSampling().fit(X)
    with pytest.raises(ValueError, match="parsed input is empty"):
        with pytest.warns(UserWarning, match="Ignoring empty element on index: 0"):
            GraphletSampling(sampling={"n_samples": 2}).fit([[]])


def test_graph_kernel_dispatch():
    for name in ("GR", "graphlet_sampling"):
        gk = GraphKernel(kernel={"name": name, "k": 4, "sampling": {"n_samples": 3}}, random_state=5)
        gk.initialize()
        assert type(gk.kernel_) is GraphletSampling and gk.kernel_.k == 4
        assert gk.kernel_.random_state is gk.random_state_


def test_vectorised_oracle_classes_equal_per_sample_ones():
    """gs_oracle.classes_of_draws (used on the large GPU workloads) against the per-sample restatement."""
    X = _graphs("loops_k5_X") + _graphs("large_k5_X")
    for k in (3, 5, 6):
        a, b = np.random.RandomState(k), np.random.RandomState(k)
        for A in X:
            size, idx = _lib.gs_draw(a, [A.shape[0]], k, 30)
            assert gs_oracle.classes_of_draws(A, size, idx) == gs_oracle.graph_classes(A, k, 30, b)
