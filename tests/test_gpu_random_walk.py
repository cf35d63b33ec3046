"""RandomWalk / RandomWalkLabeled on the H100 against the reference's goldens (tests/golden/random_walk.npz) within
the per-route bounds, plus the CG iteration counts, the global-workspace variant, row blocks, device output,
determinism and symmetry."""
import json
import os
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import rw_oracle as O  # noqa: E402
from make_golden_random_walk import as_input, unflat  # noqa: E402
from grakel_b200 import RandomWalk, RandomWalkLabeled, _lib  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(HERE, "golden", "random_walk.npz"))
CASES = sorted({k.split("/")[0] for k in GOLD.files if not k.startswith("dict/")})


def case(name):
    meta = json.loads(str(GOLD[name + "/meta"]))
    X = unflat(GOLD[name + "/X_sizes"], GOLD[name + "/X_A"], GOLD[name + "/X_L"])
    Y = unflat(GOLD[name + "/Y_sizes"], GOLD[name + "/Y_A"], GOLD[name + "/Y_L"]) if name + "/Kt" in GOLD else None
    return meta, X, Y


def estimator(meta):
    return (RandomWalk if meta["cls"] == "RW" else RandomWalkLabeled)(**meta["params"])


def magnitude(est, meta, A, La, B, Lb):
    """sum of |terms| of one pair on the spectral / series routes (None: relative bound)"""
    route, fn = est._route()
    lab = meta["cls"] == "RWL"
    if route == _lib.GK_RW_SERIES and fn == _lib.GK_RW_FINITE:
        return O.series_pair(A, B, est.mu_, La if lab else None, Lb if lab else None)[1]
    if route == _lib.GK_RW_SPECTRAL:
        lam = est._lamda
        if fn == _lib.GK_RW_INV:
            f = lambda z: 1.0 / (1.0 - lam * z)
            w1, v1 = np.linalg.eigh(A)
            w2, v2 = np.linalg.eigh(B)
            return O.spectral_pair(v1.sum(0), w1, v2.sum(0), w2, f)[1]
        f = (lambda z: np.exp(lam * z)) if fn == _lib.GK_RW_EXP else None
        if f is None:
            mu = est.mu_

            def f(z):
                D, S = np.ones_like(z), mu[0] * np.ones_like(z)
                for c in mu[1:]:
                    D = D * z
                    S = S + c * D
                return S
        return O.spectral_pair(*O.eig_data(A), *O.eig_data(B), f)[1]
    return None


def check(est, meta, K, ref, rows, cols, drows, dcols):
    route, fn = est._route()
    rel = 1e-10 if route == _lib.GK_RW_CG else 1e-11
    norm = bool(meta["params"].get("normalize"))
    for i in range(K.shape[0]):
        for j in range(K.shape[1]):
            (A, La), (B, Lb) = rows[i], cols[j]
            mag = magnitude(est, meta, A, La, B, Lb)
            if mag is None:
                tol = rel * abs(ref[i, j]) * (3 if norm else 1)
            else:
                tol = 1e-12 * mag * (3 if norm else 1)
                if norm:
                    tol /= np.sqrt(abs(drows[i] * dcols[j]))
            assert abs(K[i, j] - ref[i, j]) <= tol, (i, j, K[i, j], ref[i, j], tol)


@pytest.mark.parametrize("name", CASES)
def test_golden(name):
    meta, X, Y = case(name)
    est = estimator(meta)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        K = est.fit_transform(as_input(X))
        Kt = est.transform(as_input(Y)) if Y is not None else None
    msgs = [str(x.message) for x in w if issubclass(x.category, RuntimeWarning)]
    assert msgs == meta["warnings"] and est._lamda == meta["lamda_used"]
    assert np.array_equal(K, K.T)
    dx = est._X_diag
    check(est, meta, K, GOLD[name + "/K"], X, X, dx, dx)
    if Y is not None:
        check(est, meta, Kt, GOLD[name + "/Kt"], Y, X, est._Y_diag, dx)


@pytest.mark.parametrize("name", ["mutag_rw_test_lamda", "mutag_rwl_default", "directed_signed_cg_labeled",
                                  "empty_label_intersection"])
def test_cg_iterations(name):
    meta, X, _ = case(name)
    est = estimator(meta)
    est.fit_transform(as_input(X))
    its = _lib.get_engine().rw_iterations(len(X), len(X))
    lab = meta["cls"] == "RWL"
    for i in range(len(X)):
        for j in range(len(X)):
            a, b = X[min(i, j)], X[max(i, j)]
            _, it = O.cg_pair(a[0], b[0], est._lamda, a[1] if lab else None, b[1] if lab else None)
            assert its[i, j] == it, (i, j)


def test_global_workspace_pair():
    rs = np.random.RandomState(7)
    G = []
    for n in (100, 12, 95):  # 3 x 8 x 100 x 100 bytes exceed a CTA's shared memory
        A = np.triu((rs.rand(n, n) < 0.05).astype(float), 1)
        G.append((A + A.T, [int(x) for x in rs.randint(2, size=n)]))
    for cls in (RandomWalk, RandomWalkLabeled):
        K = cls(lamda=0.01).fit_transform(as_input(G))
        lab = cls is RandomWalkLabeled
        for i in range(3):
            for j in range(i, 3):
                v, _ = O.cg_pair(G[i][0], G[j][0], 0.01, G[i][1] if lab else None, G[j][1] if lab else None)
                assert abs(K[i, j] - v) <= 1e-10 * abs(v)


@pytest.mark.parametrize("params", [dict(lamda=0.02), dict(lamda=0.1, p=3, method_type="baseline"),
                                    dict(lamda=0.2, kernel_type="exponential")], ids=str)
def test_rows_device_output_determinism(params):
    torch = pytest.importorskip("torch")
    meta, X, _ = case("directed_signed_cg")
    est = RandomWalk(**params)
    K1 = est.fit_transform(as_input(X + X[:3]))
    K2 = est.fit_transform(as_input(X + X[:3]))
    assert np.array_equal(K1, K2) and np.array_equal(K1, K1.T)
    n = K1.shape[0]
    eng = _lib.get_engine()
    Kb, _, _ = eng.gram(n, row_range=(2, 7))
    assert np.array_equal(Kb, K1[2:7])
    t = torch.full((n, n), float("nan"), dtype=torch.float64, device="cuda")
    eng.gram(n, device_ptr=t.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), K1)
    Kn = RandomWalk(normalize=True, **params).fit_transform(as_input(X + X[:3]))
    d = np.diag(K1)
    with np.errstate(invalid="ignore"):
        assert np.allclose(Kn, K1 / np.sqrt(np.outer(d, d)), rtol=1e-14, atol=0, equal_nan=True)


def test_read_tu_block_equals_list():
    """A read_tu(kernel="SP") block walks the nodes that occur in an edge, as the reference's edge dictionaries do."""
    import tempfile
    import make_golden_neighborhood_hash as mg
    from make_golden_tu import unpack
    from grakel_b200.datasets import read_tu
    d = tempfile.mkdtemp()
    unpack("MUTAG", d)
    block = read_tu(d, "MUTAG", kernel="SP").data
    X = mg.mutag()
    for cls, lam in ((RandomWalk, 0.01), (RandomWalkLabeled, 1e-4)):
        Kb = cls(lamda=lam).fit_transform(block)
        Kl = cls(lamda=lam).fit_transform(X)
        assert np.allclose(Kb, Kl, rtol=1e-12, atol=0)
