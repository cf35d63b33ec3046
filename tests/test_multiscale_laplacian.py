"""MultiscaleLaplacian on the host: the Cholesky oracle against the reference's goldens, the reference's samples,
parameter validation, the deviations that raise NotImplementedError before any device work, GraphKernel dispatch."""
import warnings

import numpy as np
import pytest

from grakel_b200 import GraphKernel, MultiscaleLaplacian
from ml_cases import ERROR_CASES, as_input, load, rel_err, replay_eig
from ml_oracle import MLOracle

META, CASES = load()
BAR = 1e-9


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_golden(name):
    c = CASES[name]
    g = c["g"]
    for norm in (False, True):
        o = MLOracle(eig=replay_eig(g, c["levels"]), **c["params"])
        K = o.fit_transform(c["X"], normalize=norm)
        assert rel_err(K, g["K_fit" + ("_norm" if norm else "")]) <= BAR
        assert rel_err(o.transform(c["Y"], normalize=norm), g["K_tr" + ("_norm" if norm else "")]) <= BAR
        for l, vs in enumerate(o.samples):
            assert [(k, j) for k, j in g["samples_%d" % l]] == vs


def test_oracle_own_eig_on_reference_tests():
    c = CASES["reference_tests"]
    o = MLOracle(**c["params"])
    assert rel_err(o.fit_transform(c["X"]), c["g"]["K_fit"]) <= BAR
    assert rel_err(o.transform(c["Y"]), c["g"]["K_tr"]) <= BAR


@pytest.mark.parametrize("name", sorted(META["errors"]))
def test_validation_errors(name):
    params = dict(ERROR_CASES)[name]
    X = as_input(CASES["weighted_loops"]["X"])
    if name == "int_labels":
        X = [[A, {i: 1 for i in range(len(A))}] for A, _ in X]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception) as e:
            MultiscaleLaplacian(**params).fit_transform(X)
    assert type(e.value).__name__ == META["errors"][name]


def _graph(n, seed=0):
    rs = np.random.RandomState(seed)
    A = np.triu((rs.rand(n, n) < 0.3).astype(float), 1)
    return A + A.T, rs.rand(n, 3)


@pytest.mark.parametrize("case", ["non_symmetric", "negative_weight", "gamma_zero", "heta_zero", "too_large"])
def test_deviations_raise(case):
    A, phi = _graph(8)
    params = {}
    if case == "non_symmetric":
        A[0, 1], A[1, 0] = 1.0, 0.0
    elif case == "negative_weight":
        A[0, 1] = A[1, 0] = -1.0
    elif case == "gamma_zero":
        params = dict(gamma=0.0)
    elif case == "heta_zero":
        params = dict(heta=0.0)
    else:
        A, phi = _graph(129)
    X = as_input([(A, phi), _graph(5, 1)])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(NotImplementedError):
            MultiscaleLaplacian(**params).fit_transform(X)


def test_graph_kernel_dispatch():
    gk = GraphKernel(kernel="ML", random_state=5)
    gk.initialize()
    cls, params = gk.make_kernel_(["ML"], {})
    assert cls is MultiscaleLaplacian and params["random_state"] is gk.random_state_
    gk = GraphKernel(kernel="multiscale_laplacian", random_state=5)
    gk.initialize()
    assert gk.make_kernel_(["multiscale_laplacian"], {})[0] is MultiscaleLaplacian


def test_read_tu_block_without_attributes(tmp_path):
    """A datasets.read_tu block without node attributes has no features: the reference's TypeError, before any
    device work."""
    import copy
    from make_golden_tu import unpack
    from grakel_b200.datasets import read_tu
    unpack("Cuneiform", str(tmp_path))
    block = copy.copy(read_tu(str(tmp_path), "Cuneiform", kernel="SP", prefer_attr_nodes=True).data)
    block.attrs = None
    with pytest.raises(TypeError, match="Features must be iterable"):
        MultiscaleLaplacian().fit_transform(block)
