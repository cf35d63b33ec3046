"""SubgraphMatching on the device: bit for bit against the real reference's goldens, per-pair counts against the
oracle, and the routes (row ranges, device output, records read from global memory) against each other."""
import json
import os
import sys
from math import comb, factorial

import numpy as np
import pytest

from grakel_b200 import Graph, GraphKernel, SubgraphMatching
from grakel_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sm_oracle  # noqa: E402
from nspd_cases import _rand_graph, mutag  # noqa: E402
from sm_cases import GRAPH_OBJECT_CASES, cases  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "subgraph_matching.npz"))
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
    k = SubgraphMatching(normalize=bool(norm), **p)
    K = k.fit_transform(X)
    ref = G[f"{name}/fit/{norm}"]
    assert K.shape == ref.shape and np.array_equal(K, ref, equal_nan=True), np.nanmax(np.abs(K - ref))
    if Y is not None:
        Kt = k.transform(Y)
        ref = G[f"{name}/transform/{norm}"]
        assert Kt.shape == ref.shape and np.array_equal(Kt, ref, equal_nan=True), np.nanmax(np.abs(Kt - ref))


def _counts(k, graphs, n_fit, row):
    gp, rp, ci, ids, elids, vt, et, flags = k._pack(graphs)
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, ids, None, None)
        eng.sm_features(int(k.k), k.lambdas_, vt, et, elids, flags)
        return eng.sm_counts(n_fit, row)


@pytest.mark.parametrize("directed", [False, True])
def test_counts_match_oracle(directed):
    rng = np.random.default_rng(21 + directed)
    X = [_rand_graph(rng, int(rng.integers(4, 11)), 0.4, 3, 2, directed=directed) for _ in range(8)]
    k = SubgraphMatching(k=6)
    k.fit(X)
    for row in range(len(X)):
        tv = _counts(k, k.X, len(X), row)
        for c in range(len(X)):
            x, y = (k.X[row], k.X[c]) if row <= c else (k.X[c], k.X[row])
            ref = [float(t) for t in sm_oracle.counts(x, y, k.kv, k.ke, 6)]
            assert np.array_equal(tv[c], ref), (row, c, tv[c], ref)


def _ke_real(a, b):
    return 0.1 + 0.37 * a + 0.11 * b


def _kv_real(a, b):
    return 1.3 if a == b else 0.7 * ((a + b) % 2)


def test_real_tables_within_bound():
    rng = np.random.default_rng(4)
    X = [_rand_graph(rng, int(rng.integers(4, 10)), 0.4, 3, 3) for _ in range(6)]
    k = SubgraphMatching(kv=_kv_real, ke=_ke_real, lw="decreasing")
    K = k.fit_transform(X)
    lam = k.lambdas_.ravel()
    for i in range(len(X)):
        for j in range(i, len(X)):
            exact = sm_oracle.counts(k.X[i], k.X[j], k.kv, k.ke, 5)
            absum = sm_oracle.counts(k.X[i], k.X[j], k.kv, k.ke, 5, absolute=True)
            ref = float(sum(l * t for l, t in zip(lam, exact)))
            bound = 1e-12 * float(sum(abs(l) * t for l, t in zip(lam, absum)))
            assert abs(K[i, j] - ref) <= bound and K[j, i] == K[i, j], (i, j, K[i, j], ref)


def test_routes_agree(monkeypatch):
    X, Y, p = CASES["mutag_k5"]
    k = SubgraphMatching(**p)
    K = k.fit_transform(X)
    assert np.array_equal(K, G["mutag_k5/fit/0"])
    assert np.array_equal(k.fit_transform(X), K)  # two runs
    Kr, _, _ = k._sm_run(k.X, len(X), row_range=(7, 31))
    assert np.array_equal(Kr, K[7:31])
    Kt = k.transform(Y)
    Kt2, _, _ = k._sm_run(k.X + k.parse_input(Y), len(X), row_range=(2, 6))
    assert np.array_equal(Kt2, Kt[2:6])
    import torch
    dev = torch.zeros((len(X), len(X)), dtype=torch.float64, device="cuda")
    k._sm_run(k.X, len(X), device_ptr=dev.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), K)
    monkeypatch.setenv("GRAKEL_B200_SM_GLOBAL", "1")
    assert np.array_equal(SubgraphMatching(**p).fit_transform(X), K)
    assert np.array_equal(SubgraphMatching(**p).fit(X).transform(Y), Kt)


def test_exact_above_2_24():
    """Two complete graphs on 11 vertices: the size-s cliques are the partial injective maps, C(11, s)^2 s! of them;
    at s = 5 that is 25 613 280 > 2^24."""
    n = 11
    g = [{i: {j: 1 for j in range(n) if j != i} for i in range(n)}, {i: 0 for i in range(n)}, {}]
    k = SubgraphMatching(kv=None, ke=None, k=5)
    k.fit([g])
    tv = _counts(k, k.X, 1, 0)[0]
    ref = [comb(n, s) ** 2 * factorial(s) for s in range(1, 6)] + [0]
    assert ref[4] > 2 ** 24 and np.array_equal(tv, np.array(ref, dtype=np.float64))
    assert k.fit_transform([g])[0, 0] == sum(ref)


def test_read_tu_block():
    import tempfile
    sys.path.insert(0, os.path.join(HERE, "golden"))
    from make_golden_tu import unpack
    from grakel_b200.datasets import read_tu
    d = tempfile.mkdtemp()
    unpack("MUTAG", d)
    tu = read_tu(d, "MUTAG", kernel="SP")
    graphs = [[ed, nl, {}] for ed, nl, _ in mutag()]
    k = SubgraphMatching(ke=None, k=4)
    assert np.array_equal(k.fit_transform(tu.data), SubgraphMatching(ke=None, k=4).fit_transform(graphs))
    # with its edge labels, the whole read_tu result gives the reference's K of the graph list
    assert np.array_equal(SubgraphMatching(k=3).fit_transform(tu), G["mutag_k3/fit/0"])


def _star(n, inward):
    """A directed star on n vertices: every edge points to (inward) or from vertex 0, so each out-degree (inward) or
    in-degree is at most 1 while vertex 0 has n - 1 neighbours."""
    ed = {i: {} for i in range(n)}
    for i in range(1, n):
        if inward:
            ed[i][0] = 1
        else:
            ed[0][i] = 1
    return [ed, {i: 0 for i in range(n)}, {(u, v): 0 for u in ed for v in ed[u]}]


@pytest.mark.parametrize("inward", [True, False])
def test_directed_hub_counts(inward):
    """The extension sets grow through out- and in-neighbours: a hub whose edges all point inward has small
    out-degrees but many c-neighbours."""
    X = [_star(10, inward), _star(7, not inward), _rand_graph(np.random.default_rng(2), 9, 0.3, 1, 1, directed=True)]
    for kk in (2, 5):
        k = SubgraphMatching(k=kk)
        k.fit(X)
        for row in range(len(X)):
            tv = _counts(k, k.X, len(X), row)
            for c in range(len(X)):
                x, y = (k.X[row], k.X[c]) if row <= c else (k.X[c], k.X[row])
                ref = [float(t) for t in sm_oracle.counts(x, y, k.kv, k.ke, kk)]
                assert np.array_equal(tv[c], ref), (kk, row, c, tv[c], ref)


def test_graphkernel_and_unsupported():
    X, _, p = CASES["random"]
    assert np.array_equal(GraphKernel(kernel={"name": "SM"}).fit_transform(X), G["random/fit/0"])
    k = SubgraphMatching()
    k.fit(X)
    gp, rp, ci, ids, elids, vt, et, flags = k._pack(k.X)
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, ids, None, None)
        eng.sm_features(int(k.k), k.lambdas_, vt, et, elids, flags)
        with pytest.raises(NotImplementedError, match="GK_DIST with SubgraphMatching features"):
            eng.gram(len(X), dist=True)
    with pytest.raises(NotImplementedError):
        SubgraphMatching(k=15, lw="decreasing").fit_transform(X)
