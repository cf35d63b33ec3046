"""NeighborhoodSubgraphPairwiseDistance on the device, bit for bit against the real reference's goldens."""
import json
import os
import sys

import numpy as np
import pytest

from grakel_b200 import Graph, GraphKernel, NeighborhoodSubgraphPairwiseDistance
from grakel_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from nspd_cases import GRAPH_OBJECT_CASES, cases  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nspd.npz"))
CASES = {}
for _name, _X, _Y, _p in cases():
    if _name in GRAPH_OBJECT_CASES:
        _X = [Graph(*x) for x in _X]
        _Y = None if _Y is None else [Graph(*y) for y in _Y]
    CASES[_name] = (_X, _Y, _p)


@pytest.mark.parametrize("name", json.loads(str(G["__cases__"])))
@pytest.mark.parametrize("norm", [0, 1])
def test_golden(name, norm):
    X, Y, p = CASES[name]
    k = NeighborhoodSubgraphPairwiseDistance(normalize=bool(norm), **p)
    K = k.fit_transform(X)
    ref = G[f"{name}/fit/{norm}"]
    assert K.shape == ref.shape and np.array_equal(K, ref), np.abs(K - ref).max()
    assert np.array_equal(K, K.T)
    if Y is not None:
        Kt = k.transform(Y)
        ref = G[f"{name}/transform/{norm}"]
        assert Kt.shape == ref.shape and np.array_equal(Kt, ref), np.abs(Kt - ref).max()


@pytest.mark.parametrize("name", json.loads(str(G["__cases__"])))
def test_hashes(name):
    """gk_nspd_hashes: H[rho, v] of every fitted vertex equals the reference's."""
    X, _, p = CASES[name]
    k = NeighborhoodSubgraphPairwiseDistance(**p)
    k.fit(X)
    gp, rp, ci, lab, el, sh, tokens = k._pack(k.X)
    ref = G[f"{name}/H"]
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, lab, None, None)
        eng.nspd_features(k.r, k.d, sh, el, tokens)
        for rho in range(k.r + 1):
            assert np.array_equal(eng.nspd_hashes(rho, len(lab)), ref[rho]), rho


def test_graphkernel_and_routes(monkeypatch):
    X, Y, p = CASES["random"]
    ref = G["random/fit/0"]
    K = GraphKernel(kernel={"name": "NSPD"}).fit_transform(X)
    assert np.array_equal(K, ref)
    k = NeighborhoodSubgraphPairwiseDistance()
    k.fit(X)
    Ks, _, _ = k._nspd_run(k.X, len(X), simt=True)
    assert np.array_equal(Ks, ref)
    Kr, _, _ = k._nspd_run(k.X, len(X), row_range=(3, 9))
    assert np.array_equal(Kr, ref[3:9])
    import torch
    dev = torch.zeros((len(X), len(X)), dtype=torch.float64, device="cuda")
    k._nspd_run(k.X, len(X), device_ptr=dev.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), ref)
    monkeypatch.setenv("GRAKEL_B200_NSPD_WS_BUDGET", "4096")
    monkeypatch.setenv("GRAKEL_B200_NSPD_C_BUDGET", "256")
    assert np.array_equal(NeighborhoodSubgraphPairwiseDistance().fit_transform(X), ref)


def test_exact_above_2_24():
    def g(n):
        return [{i: {i: 1} for i in range(n)}, {i: 0 for i in range(n)}, {(i, i): 0 for i in range(n)}]
    K = NeighborhoodSubgraphPairwiseDistance(r=0, d=0).fit_transform([g(4101), g(4099)])
    assert np.array_equal(K, np.ones((2, 2)))


def test_dist_unsupported():
    X, _, _ = CASES["random"]
    k = NeighborhoodSubgraphPairwiseDistance()
    k.fit(X)
    gp, rp, ci, lab, el, sh, tokens = k._pack(k.X)
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, lab, None, None)
        eng.nspd_features(k.r, k.d, sh, el, tokens)
        with pytest.raises(NotImplementedError, match="GK_DIST with NeighborhoodSubgraphPairwiseDistance features"):
            eng.gram(len(X), dist=True)
