"""SubgraphMatching on the host: the oracle against the reference's goldens, the lambda fold against np.dot, the
estimator's parameter checks, errors and dispatch (no GPU needed)."""
import json
import os
import sys
import warnings

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sm_oracle  # noqa: E402
from sm_cases import GRAPH_OBJECT_CASES, cases, error_cases  # noqa: E402

from grakel_b200 import Graph, GraphKernel, SubgraphMatching  # noqa: E402
from grakel_b200.kernels import _dirac  # noqa: E402

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "subgraph_matching.npz"))
# oracle rows of the large MUTAG cases: a leading block of the fitted graphs (its K is that block of the golden K)
PREFIX = {"mutag_k3": 25, "mutag_k5": 12}


def _case(name):
    return next(c for c in cases() if c[0] == name)


@pytest.mark.parametrize("name", [c[0] for c in cases()])
def test_oracle_matches_golden(name):
    _, X, Y, params = _case(name)
    if name in GRAPH_OBJECT_CASES:
        X, Y = [Graph(*x) for x in X], [Graph(*y) for y in Y]
    est = SubgraphMatching(**params)
    est.initialize()
    px = est.parse_input(X)
    pre = PREFIX.get(name)
    kv, ke, k = est.kv, est.ke, int(est.k)
    kvf = None if kv is None else kv
    kef = None if ke is None else ke
    for norm in (0, 1):
        gold = GOLD[f"{name}/fit/{norm}"]
        xs = px[:pre] if pre else px
        K = sm_oracle.gram(xs, None, kvf, kef, k, est.lambdas_, normalize=bool(norm))
        np.testing.assert_array_equal(K, gold[:len(xs), :len(xs)])
        if Y is not None and not pre:
            K = sm_oracle.gram(px, est.parse_input(Y), kvf, kef, k, est.lambdas_, normalize=bool(norm))
            np.testing.assert_array_equal(K, GOLD[f"{name}/transform/{norm}"])


def test_lambda_fold_is_np_dot():
    rng = np.random.default_rng(3)
    for n in range(1, 16):
        for _ in range(200):
            lam = rng.random(n) * 10.0 ** rng.integers(-3, 3)
            tv = np.floor(rng.random(n) * 10.0 ** rng.integers(0, 8))
            assert sm_oracle.fma_fold(lam, tv) == np.dot(lam.reshape(1, n), tv)[0]


@pytest.mark.parametrize("name", [e[0] for e in error_cases()])
def test_errors_match_golden(name):
    want = json.loads(str(GOLD["__errors__"]))[name]
    _, X, params = next(e for e in error_cases() if e[0] == name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception) as info:
            est = SubgraphMatching(**params)
            est.initialize()
            est.parse_input(X)
    assert type(info.value).__name__ == want


def test_parameters_and_dispatch():
    est = SubgraphMatching()
    assert est.kv is _dirac and est.ke is _dirac and est.k == 5 and est.lw == "uniform"
    est.initialize()
    assert est.lambdas_.shape == (1, 6)
    est = SubgraphMatching(k=0)
    est.initialize()
    assert est.lambdas_.shape == (1, 1)
    gk = GraphKernel(kernel={"name": "SM", "k": 3})
    gk.initialize()
    assert isinstance(gk.kernel_, SubgraphMatching) and gk.kernel_.k == 3
    gk = GraphKernel(kernel="subgraph_matching")
    gk.initialize()
    assert isinstance(gk.kernel_, SubgraphMatching)
    with pytest.raises(NotImplementedError):
        SubgraphMatching(k=-1).initialize()


def test_custom_kernel_table_cap():
    X = [[{0: {1: 1}, 1: {0: 1}}, {0: i, 1: i + 100}, {(0, 1): 0, (1, 0): 0}] for i in range(40)]
    est = SubgraphMatching(kv=lambda a, b: 1)
    est.initialize()
    with pytest.raises(NotImplementedError):
        est._pack(est.parse_input(X))


def test_labels_compare_by_python_equality():
    est = SubgraphMatching()
    est.initialize()
    g = est.parse_input([[{0: {1: 1}, 1: {0: 1}}, {0: 1, 1: 1.0}, {(0, 1): True, (1, 0): 1}]])
    _, _, ids, elids, _, _, _ = est._pack(g)[1:]
    assert len(set(ids.tolist())) == 1 and len(set(elids.tolist())) == 1


def test_read_tu_result_parses_as_its_graphs():
    import tempfile
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    from make_golden_tu import unpack
    from nspd_cases import mutag
    from grakel_b200.datasets import read_tu
    d = tempfile.mkdtemp()
    unpack("MUTAG", d)
    tu = read_tu(d, "MUTAG", kernel="SP")
    est = SubgraphMatching()
    est.initialize()
    assert est.parse_input(tu) == est.parse_input(mutag())
    with pytest.raises(NotImplementedError):
        est.parse_input(tu.data)
    est = SubgraphMatching(ke=None)
    est.initialize()
    assert est.parse_input(tu.data) == est.parse_input([[ed, nl, {}] for ed, nl, _ in mutag()])
