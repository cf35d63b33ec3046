"""PyramidMatch and WeisfeilerLehman over it on the device, fed the reference's golden embeddings through the
`eigs` / `eig` seam: every level's cells and K of fit_transform / transform bit for bit against the goldens; on
generated graphs against the NumPy restatement, with row blocks, device output, normalisation, exact symmetry,
determinism and the chunked level Grams."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import pm_oracle  # noqa: E402
from grakel_b200 import GraphKernel, PyramidMatch, WeisfeilerLehman, _lib, kernels  # noqa: E402
from test_pyramid_match import CASES, GOLDEN, INPUTS, WL_CASES, WL_INPUTS, golden_calls, mg, raw_labels  # noqa: E402

pytestmark = pytest.mark.gpu


class Replay:
    """eigs / eig that hand out given |U| in call order: eigenvalues in descending order, so the reference's
    argsort()[::-1] keeps the columns, and absolute() keeps the values."""

    def __init__(self, calls):
        self.calls = list(calls)
        self.i = 0

    def _next(self):
        u = self.calls[self.i]
        self.i += 1
        return u

    def eigs(self, A, k, ncv):
        u = self._next()
        return np.arange(u.shape[1], 0, -1).astype(float), u

    def eig(self, A):
        u = self._next()
        n = A.shape[0]
        return np.arange(n, 0, -1).astype(float), np.pad(u, ((0, 0), (0, n - u.shape[1])))


@pytest.fixture
def replay(monkeypatch):
    def use(calls):
        r = Replay(calls)
        monkeypatch.setattr(kernels, "eigs", r.eigs)
        monkeypatch.setattr(kernels, "eig", r.eig)
        return r
    return use


def _same(a, b):
    assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("name,spec", CASES, ids=lambda x: str(x))
def test_golden_cases(name, spec, replay):
    X, Y, _ = INPUTS[name]
    wl, L, d, norm, _ = spec
    key = mg.case_key(name, spec)
    r = replay(golden_calls(key))
    est = PyramidMatch(with_labels=wl, L=L, d=d, normalize=norm)
    _same(est.fit_transform(X), GOLDEN[key + "__K_fit"])
    _same(est.transform(Y), GOLDEN[key + "__K_tr"])
    assert r.i == len(r.calls)


@pytest.mark.parametrize("name,spec", [c for c in CASES if c[1][1] > 0][:6], ids=lambda x: str(x))
def test_golden_cells(name, spec, replay):
    X, Y, _ = INPUTS[name]
    wl, L, d, norm, _ = spec
    us = golden_calls(mg.case_key(name, spec))
    replay(us)
    est = PyramidMatch(with_labels=wl, L=L, d=d).fit(X)
    data = est.X
    with _lib.engine() as eng:
        gp = np.concatenate([[0], np.cumsum(data.sizes)])
        V = int(gp[-1])
        eng.pack(gp, np.zeros(V + 1, dtype=np.int32), np.zeros(0, dtype=np.int32),
                 est._label_ids(data, len(data)) if wl else None, None, None)
        eng.pm_features(L, d, data.U, data.n_cols, flags=_lib.GK_PM_LABELS if wl else 0)
        for j in range(L):
            cells = eng.pm_cells(0, j, V, d)
            want = np.full((V, d), -1, dtype=np.int64)
            for g, u in enumerate(us[:len(X)]):
                T = np.floor(u * 2 ** j)
                T[T == 2 ** j] = 2 ** j - 1
                want[gp[g]:gp[g + 1], :u.shape[1]] = T
            assert np.array_equal(cells, want)


@pytest.mark.parametrize("name,spec", WL_CASES, ids=lambda x: str(x))
def test_wl_golden_cases(name, spec, replay):
    X, Y, _ = WL_INPUTS[name]
    h, wl, L, d, norm, _ = spec
    key = mg.case_key(name, spec)
    r = replay(golden_calls(key))
    est = WeisfeilerLehman(n_iter=h, normalize=norm,
                           base_graph_kernel=(PyramidMatch, {"with_labels": wl, "L": L, "d": d}))
    _same(est.fit_transform(X), GOLDEN[key + "__K_fit"])
    _same(est.transform(Y), GOLDEN[key + "__K_tr"])
    assert r.i == len(r.calls)


@pytest.mark.parametrize("name,spec", WL_CASES, ids=lambda x: str(x))
def test_wl_golden_cases_with_reordered_label_dicts(name, spec, replay):
    """The labels dictionaries' key order fixes the packed vertex order, not K: reversed dictionaries give the
    reference's K (wl_iso also labels vertices outside the edge dictionary, which the base kernel does not see)."""
    X, Y, _ = WL_INPUTS[name]
    h, wl, L, d, norm, _ = spec
    key = mg.case_key(name, spec)
    rev = lambda G: [[x[0], dict(reversed(list(x[1].items())))] for x in G]  # noqa: E731
    replay(golden_calls(key))
    est = WeisfeilerLehman(n_iter=h, normalize=norm,
                           base_graph_kernel=(PyramidMatch, {"with_labels": wl, "L": L, "d": d}))
    _same(est.fit_transform(rev(X)), GOLDEN[key + "__K_fit"])
    _same(est.transform(rev(Y)), GOLDEN[key + "__K_tr"])


def test_embedding_values_out_of_range_are_refused():
    """gk_pm_features takes |U| in [0, 1 + 2^-(L-1)): a NaN, a negative value or one past the last cell is GK_ERR_ARG."""
    gp = np.array([0, 3])
    for bad in (np.nan, -0.25, 1.5):
        U = np.full((1, 3, 2), 0.5)
        U[0, 1, 1] = bad
        with _lib.engine() as eng:
            eng.pack(gp, np.zeros(4, dtype=np.int32), np.zeros(0, dtype=np.int32), None, None, None)
            with pytest.raises(_lib.GrakelB200Error, match="embedding value"):
                eng.pm_features(3, 2, U, np.array([[2]]))
            U[0, 1, 1] = 1.0 + 2.0 ** -3  # the largest cell clamps; a skipped vertex is not looked at
            skip = np.array([0, 0, 0], dtype=np.uint8)
            eng.pm_features(3, 2, U, np.array([[2]]), skip=skip)
            U[0, 1, 1] = bad
            eng.pm_features(3, 2, U, np.array([[2]]), skip=np.array([0, 1, 0], dtype=np.uint8))


def test_graph_kernel_goldens(replay):
    mu = mg.mutag()[:20]
    for key, kernel in (("gk_pm", {"name": "PM", "L": 3, "d": 4}),
                        ("gk_wl_pm", [{"name": "WL", "n_iter": 2}, {"name": "pyramid_match", "d": 4}])):
        replay(golden_calls(key))
        _same(GraphKernel(kernel=kernel, normalize=True).fit_transform(mu), GOLDEN[key + "__K_fit"])


# ---- generated graphs: the device against the restatement and against itself
def _gen(n, seed=0):
    sys.path.insert(0, os.path.join(HERE, ".."))
    import bench
    return bench.gen_list(n, 40, seed)


@pytest.fixture(scope="module")
def fitted():
    import warnings
    warnings.simplefilter("ignore")
    X = _gen(2400)
    est = PyramidMatch(L=4, d=6).fit(X)
    return X, est


def _oracle_rows(est, rows, n_cols=None):
    data = est.X
    gp = np.concatenate([[0], np.cumsum(data.sizes)])
    us = [data.U[0, gp[g]:gp[g + 1], :data.n_cols[0, g]] for g in range(len(data))]
    labels = [[est._labels[l] for l in data.labels[gp[g]:gp[g + 1]]] for g in range(len(data))]
    H = pm_oracle.histograms(us, labels, est.L, est.d, len(est._labels) * est.d)
    cols = range(len(data)) if n_cols is None else range(n_cols)
    return np.array([[pm_oracle.pair(H[i], H[j], est.L) for j in cols] for i in rows])


def test_against_restatement(fitted):
    X, est = fitted
    K, _, _ = est._pm_run(est.X, len(est.X))
    assert np.array_equal(K, K.T)
    rows = list(range(0, len(X), 97))
    assert np.array_equal(K[rows], _oracle_rows(est, rows))


def test_variants_equal_the_full_matrix(fitted, monkeypatch):
    import torch
    X, est = fitted
    data, n = est.X, len(est.X)
    full, xd, _ = est._pm_run(data, n)
    again, _, _ = est._pm_run(data, n)
    assert np.array_equal(full, again)
    assert np.array_equal(xd, np.diagonal(full))
    gp = np.concatenate([[0], np.cumsum(data.sizes)])
    V = int(gp[-1])
    ids = est._label_ids(data, n)
    with _lib.engine() as eng:
        eng.pack(gp, np.zeros(V + 1, dtype=np.int32), np.zeros(0, dtype=np.int32), ids, None, None)
        eng.pm_features(est.L, est.d, data.U, data.n_cols, flags=_lib.GK_PM_LABELS)
        blk, _, _ = eng.gram(n, row_range=(300, 1234))
        assert np.array_equal(blk, full[300:1234])
        out = torch.full((n, n + 3), float("nan"), dtype=torch.float64, device="cuda")
        eng.gram(n, device_ptr=out.data_ptr(), ld=n + 3)
        torch.cuda.synchronize()
        assert np.array_equal(out[:, :n].cpu().numpy(), full)
        Kn, _, _ = eng.gram(n, normalize=True)
        with np.errstate(invalid="ignore", divide="ignore"):
            assert np.array_equal(Kn, full / np.sqrt(np.outer(xd, xd)))
        Kt, xd2, yd = eng.gram(n, n_fit=2000)
        assert np.array_equal(Kt, full[2000:, :2000])
        assert np.array_equal(xd2, xd[:2000]) and np.array_equal(yd, xd[2000:])
        monkeypatch.setenv("GRAKEL_B200_NH_C_BUDGET", str(4 * 2400 * 300 * 4))  # about 300 rows per chunk
        Kc, _, _ = eng.gram(n)
        assert np.array_equal(Kc, full)
        with pytest.raises(NotImplementedError):
            eng.gram(n, dist=True)


def test_transform_against_restatement(replay):
    X, Y = _gen(300, 1), _gen(40, 2)
    est = PyramidMatch(L=4, d=6, normalize=True)
    K = est.fit_transform(X)
    Kt = est.transform(Y)
    data = est.X
    gp = np.concatenate([[0], np.cumsum(data.sizes)])
    us = [data.U[0, gp[g]:gp[g + 1], :data.n_cols[0, g]] for g in range(len(data))]
    est._method_calling = 3
    Yd = est.parse_input(Y)  # a second embedding of Y: compare through the restatement of this one
    gy = np.concatenate([[0], np.cumsum(Yd.sizes)])
    uy = [Yd.U[0, gy[g]:gy[g + 1], :Yd.n_cols[0, g]] for g in range(len(Yd))]
    replay(us + uy)
    est2 = PyramidMatch(L=4, d=6, normalize=True)
    est2.fit(X)
    Kt2 = est2.transform(Y)
    lx = raw_labels(X)
    ly = raw_labels(Y)
    Ko, Kto = pm_oracle.kernel(us, 4, 6, lx, uy, ly, normalize=True)
    assert np.array_equal(K, Ko)
    assert np.array_equal(Kt2, Kto)
    assert Kt.shape == Kto.shape
