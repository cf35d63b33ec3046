"""gk_gram's request contract, route by route: row blocks, pitched host output, device output, the self similarities,
normalisation, and the refusals of each feature kind.  Every route runs on the feature block its estimator builds
for a seeded fit / transform split; Engine.gram is wrapped so that the checks run on that block."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle.gk_oracle import gen  # noqa: E402
from grakel_b200 import (GraphHopper, NeighborhoodHash, Propagation, RandomWalk, ShortestPath,  # noqa: E402
                         ShortestPathAttr, WeisfeilerLehman, _lib)
from grakel_b200._lib import GrakelB200Error  # noqa: E402

pytestmark = pytest.mark.gpu

N_FIT, N_Y = 30, 12


def _attributed(seed, signed):
    X = gen(N_FIT + N_Y, 9, seed, attr=3, as_adj=True)
    if signed:
        for _, L in X:
            for v in L:
                L[v] = L[v] - 0.5
    return X


# route -> (estimator, input, fp32 output, device output, row map, GK_DIST, normalises)
ROUTES = {
    "wl": (lambda: WeisfeilerLehman(n_iter=3), lambda: gen(N_FIT + N_Y, 10, 1), True, True, True, True, True),
    "sp": (lambda: ShortestPath(), lambda: gen(N_FIT + N_Y, 10, 2, as_adj=True), True, True, True, True, True),
    "pk": (lambda: Propagation(random_state=0), lambda: gen(N_FIT + N_Y, 10, 3), True, True, False, False, True),
    "spattr_tf32": (lambda: ShortestPathAttr(), lambda: _attributed(4, False), False, False, False, False, True),
    "spattr_f64": (lambda: ShortestPathAttr(), lambda: _attributed(5, True), False, False, False, False, True),
    "gh_linear": (lambda: GraphHopper(kernel_type="linear"), lambda: _attributed(6, False), False, False, False, False,
                  True),
    "gh_gaussian": (lambda: GraphHopper(kernel_type=("gaussian", 0.5)), lambda: _attributed(7, False), False, False,
                    False, False, True),
    "gh_bridge": (lambda: GraphHopper(kernel_type="bridge"), lambda: _attributed(8, False), False, False, False, False,
                  True),
    "nh_simple": (lambda: NeighborhoodHash(R=3, nh_type="simple", random_state=0), lambda: gen(N_FIT + N_Y, 10, 9),
                  False, True, False, False, False),
    "rw_cg": (lambda: RandomWalk(lamda=0.01), lambda: gen(N_FIT + N_Y, 8, 10, as_adj=True), False, True, False, False,
              True),
    "rw_spectral": (lambda: RandomWalk(lamda=0.01, kernel_type="exponential"),
                    lambda: gen(N_FIT + N_Y, 8, 11, as_adj=True), False, True, False, False, True),
    "rw_series": (lambda: RandomWalk(lamda=0.01, method_type="baseline", p=3),
                  lambda: gen(N_FIT + N_Y, 8, 12, as_adj=True), False, True, False, False, True),
}


def _gram(eng, n, n_fit, flags=0, rows=(0, -1), K=None, dtype=_lib.GK_F64, ld=0, xd=None, yd=None):
    """gk_gram on the engine's feature block; K: host array, device pointer (int) or None."""
    kptr = C.c_void_p(K) if isinstance(K, int) else _lib._ptr(K)
    eng._check(eng.lib.gk_gram(eng.h, n_fit, flags, rows[0], rows[1], kptr, dtype, ld, _lib._ptr(xd), _lib._ptr(yd),
                               C.byref(_lib.GkStats())))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _check_route(eng, n, route):
    _, _, f32, dev, row_map, dist, normalises = ROUTES[route]
    for n_fit in (n, N_FIT):
        square = n_fit == n
        rows = n if square else n - n_fit
        K = np.empty((rows, n_fit))
        xd, yd = np.empty(n_fit), (None if square else np.empty(n - n_fit))
        _gram(eng, n, n_fit, K=K, xd=xd, yd=yd)
        if square:
            d = xd.copy()
            if route == "nh_simple":
                assert np.all(d == 1.0)
            elif route == "spattr_f64":  # the fp64 Gram sums its diagonal in another order than the self similarities
                np.testing.assert_allclose(np.diag(K), d, rtol=1e-12)
            else:
                assert np.array_equal(_bits(np.diag(K)), _bits(d))
        else:
            assert np.array_equal(_bits(xd), _bits(d[:n_fit])) and np.array_equal(_bits(yd), _bits(d[n_fit:]))

        # a row block equals the same rows of the full K
        a, b = rows // 3, rows // 3 + max(1, rows // 4)
        Kb = np.empty((b - a, n_fit))
        _gram(eng, n, n_fit, rows=(a, b), K=Kb)
        if square and route in ("spattr_tf32", "gh_linear"):
            # the 3xTF32 Gram mirrors the full square K's upper triangle; a row block computes its entries below the
            # diagonal with the operands swapped, which the split sums in another order (within its 1e-5 bound)
            upper = np.triu(np.ones((rows, n_fit), dtype=bool))[a:b]
            assert np.array_equal(_bits(Kb[upper]), _bits(K[a:b][upper])), (route, n_fit)
            np.testing.assert_allclose(Kb, K[a:b], rtol=1e-5)
        else:
            assert np.array_equal(_bits(Kb), _bits(K[a:b])), (route, n_fit)

        # pitched host output
        Kp = np.full((rows, n_fit + 3), np.nan)
        _gram(eng, n, n_fit, K=Kp, ld=n_fit + 3)
        assert np.array_equal(_bits(Kp[:, :n_fit]), _bits(K)) and np.all(np.isnan(Kp[:, n_fit:]))

        # pitched device output
        import torch
        out = torch.full((rows, n_fit + 3), float("nan"), dtype=torch.float64, device="cuda")
        if dev:
            _gram(eng, n, n_fit, flags=_lib.GK_OUT_DEVICE, K=out.data_ptr(), ld=n_fit + 3)
            torch.cuda.synchronize()
            o = out.cpu().numpy()
            assert np.array_equal(_bits(o[:, :n_fit]), _bits(K)) and np.all(np.isnan(o[:, n_fit:]))
        else:
            with pytest.raises(NotImplementedError):
                _gram(eng, n, n_fit, flags=_lib.GK_OUT_DEVICE, K=out.data_ptr(), ld=n_fit + 3)
        del out

        # normalisation by the self similarities
        Kn = np.empty_like(K)
        _gram(eng, n, n_fit, flags=_lib.GK_NORMALIZE, K=Kn)
        if normalises:
            dr = d if square else d[n_fit:]
            with np.errstate(invalid="ignore", divide="ignore"):
                ref = K / np.sqrt(np.outer(dr, d[:n_fit]))
            np.testing.assert_allclose(Kn, ref, rtol=1e-13, atol=0, equal_nan=True)
        else:
            assert np.array_equal(_bits(Kn), _bits(K))

        # fp32 output
        if f32:
            K32 = np.empty((rows, n_fit), dtype=np.float32)
            _gram(eng, n, n_fit, K=K32, dtype=_lib.GK_F32)
            assert np.array_equal(K32, K.astype(np.float32))
        else:
            with pytest.raises(NotImplementedError, match="fp64 only"):
                _gram(eng, n, n_fit, K=np.empty((rows, n_fit), dtype=np.float32), dtype=_lib.GK_F32)

        # refusals of malformed requests
        with pytest.raises(GrakelB200Error, match="bad row range"):
            _gram(eng, n, n_fit, rows=(0, rows + 1), K=np.empty((rows + 1, n_fit)))
        with pytest.raises(GrakelB200Error, match="ld smaller than the row length"):
            _gram(eng, n, n_fit, K=np.empty((rows, n_fit)), ld=n_fit - 1)
        if dist:  # the integer routes accept GK_DIST, which needs a communicator
            with pytest.raises(GrakelB200Error, match="GK_DIST without gk_comm_init"):
                _gram(eng, n, n_fit, flags=_lib.GK_DIST, K=K.copy())
        else:
            with pytest.raises(NotImplementedError, match="GK_DIST"):
                _gram(eng, n, n_fit, flags=_lib.GK_DIST, K=K.copy())

    # a row map: the identity reproduces K where it is accepted
    eng.set_row_map(n, np.arange(n, dtype=np.int32))
    try:
        Km = np.empty((n, n))
        if row_map:
            _gram(eng, n, n, K=Km)
            Ks = np.empty((n, n))
            eng.set_row_map(0, None)
            _gram(eng, n, n, K=Ks)
            assert np.array_equal(_bits(Km), _bits(Ks))
        else:
            with pytest.raises(NotImplementedError, match="row map"):
                _gram(eng, n, n, K=Km)
    finally:
        eng.set_row_map(0, None)


@pytest.mark.parametrize("route", sorted(ROUTES))
def test_gram_request_contract(route, monkeypatch):
    make, data = ROUTES[route][:2]
    X = data()
    est = make().fit(X[:N_FIT])
    gram = _lib.Engine.gram
    ran = []

    def probe(self, n_graphs, n_fit=None, **kw):
        if not ran:
            assert n_fit == N_FIT and n_graphs == N_FIT + N_Y
            _check_route(self, n_graphs, route)
            ran.append(True)
        return gram(self, n_graphs, n_fit=n_fit, **kw)

    monkeypatch.setattr(_lib.Engine, "gram", probe)
    est.transform(X[N_FIT:])
    assert ran, "the estimator's transform did not reach gk_gram"
