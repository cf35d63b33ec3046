"""SvmTheta on the device: every golden by ==, the eigenvalue bound and the float32 scale, iteration counts, the
oracle on bench.gen_list graphs, transform, normalisation, row ranges, device output, the custom-metric route, the
128-vertex cap, pickling and reruns."""
import os
import pickle
import sys
import time
import warnings

import numpy as np
import pytest

import svmt_cases
import svmt_oracle as oracle
from grakel_b200 import GraphKernel, SvmTheta, _lib

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
pytestmark = pytest.mark.gpu

Z, INPUTS = svmt_cases.load()
SEEDED = [c for c in INPUTS if c + "/xg_m" in Z]
PARAMS = {c[0]: c[3] for c in svmt_cases.cases()}
PARAMS.update(reference_tests=dict(random_state=0), mutag=dict(random_state=1),
              mutag_6_8=dict(random_state=1, subsets_size_range=(6, 8)))
wrap = lambda G: [[A] for A in G]  # noqa: E731


def _eq(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("name", SEEDED)
def test_golden(name):
    X, Y = INPUTS[name]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for norm in (0, 1):
            k = SvmTheta(normalize=bool(norm), **PARAMS[name])
            k._keep_details = True
            assert _eq(k.fit_transform(wrap(X)), Z[f"{name}/fit/{norm}"])
            if not norm:
                d = k.details_
                m = Z[name + "/xg_m"]
                assert np.all(np.abs(d["m"] - m) <= 1e-13 * np.maximum(1.0, np.abs(m)))
                shift = (m < 0) & (np.abs(m) > 1e-6)
                dev_shift = (d["m"] < 0) & (np.abs(d["m"]) > 1e-6)
                assert np.array_equal(shift, dev_shift)
                assert np.array_equal(np.float32(1.0 / -d["m"][shift]), np.float32(1.0 / -m[shift]))
                assert _eq(d["alpha"], Z[name + "/xg_alpha"])
                assert np.array_equal(d["iters"], Z[name + "/xg_iters"])
                assert _eq(np.array([x[:, 0] for x in k.X]), Z[name + "/xg_phi"])
                assert np.array_equal(d["drawn"], Z[name + "/xg_drawn"])
            assert _eq(k.transform(wrap(Y)), Z[f"{name}/transform/{norm}"])
            if not norm:
                assert _eq(k.details_["alpha"], Z[name + "/yg_alpha"])
                assert np.array_equal(k.details_["iters"], Z[name + "/yg_iters"])
                _, key, pos, _, _ = k.random_state_.get_state()
                assert np.array_equal(key, Z[name + "/state_transform_key"]) and pos == Z[name + "/state_transform_pos"]


def test_second_fit_graph_kernel_custom_metric():
    name, base, params = svmt_cases.SECOND_FIT
    X, Y = INPUTS[base]
    k = SvmTheta(**params)
    k.fit(wrap(X))
    assert _eq(k.fit_transform(wrap(X)), Z[name + "/fit/0"])
    assert _eq(k.transform(wrap(Y)), Z[name + "/transform/0"])
    for name, base, params in (svmt_cases.GRAPH_KERNEL, svmt_cases.GRAPH_KERNEL_DICT):
        X, Y = INPUTS[base]
        gk = GraphKernel(**params)
        assert _eq(gk.fit_transform(wrap(X)), Z[name + "/fit/0"])
        assert _eq(gk.transform(wrap(Y)), Z[name + "/transform/0"])
    name, base, params = svmt_cases.CUSTOM_METRIC
    X, Y = INPUTS[base]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for norm in (0, 1):
            k = SvmTheta(normalize=bool(norm), **params)
            assert _eq(k.fit_transform(wrap(X)), Z[f"{name}/fit/{norm}"])
            assert _eq(k.transform(wrap(Y)), Z[f"{name}/transform/{norm}"])


def _gen(directed=False):
    import bench
    G = [g[0] for g in bench.gen_list(200, 40, 0, as_adj=True)]
    if directed:  # keep one direction of every edge, and only graphs libsvm converges on
        rs = np.random.RandomState(1)
        out = []
        for A in G[:60]:
            D = np.triu(A) * (rs.rand(*A.shape) < 0.5)
            D = D + np.tril(A) * (D.T == 0)
            _, K = oracle.theta_matrix(D)
            if np.asarray(oracle.OneClassSVM(kernel="precomputed", max_iter=200000).fit(K).n_iter_).max() < 200000:
                out.append(D)
        G = out
    return G


@pytest.mark.parametrize("directed", [False, True])
@pytest.mark.parametrize("rng", [(2, 8), (6, 8)])
def test_gen_list_against_oracle(directed, rng):
    G = _gen(directed)
    k = SvmTheta(random_state=4, subsets_size_range=rng)
    k._keep_details = True
    o = oracle.SvmThetaOracle(random_state=4, subsets_size_range=rng)
    assert _eq(k.fit_transform(wrap(G)), o.fit_transform(G))
    _, alphas, iters = zip(*(oracle.theta_alphas(A) for A in G))
    assert _eq(k.details_["alpha"], np.concatenate(alphas))
    assert np.array_equal(k.details_["iters"], np.array(iters))
    if rng == (6, 8):
        assert np.count_nonzero(np.array([x[0, 0] for x in k.X])) > 0


def test_rows_device_output_normalize_rerun():
    import torch
    G = _gen()
    X, Y = G[:150], G[150:]
    k = SvmTheta(random_state=5, subsets_size_range=(6, 8), normalize=True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        K = k.fit_transform(wrap(X))
        Kt = k.transform(wrap(Y))
    o = oracle.SvmThetaOracle(random_state=5, subsets_size_range=(6, 8), normalize=True)
    assert _eq(K, o.fit_transform(X)) and _eq(Kt, o.transform(Y))
    xd, yd = k.diagonal()
    assert _eq(xd, o.xd)
    # row ranges and device output, fit and transform
    k = SvmTheta(random_state=6, subsets_size_range=(6, 8))
    k.initialize()
    with _lib.engine() as eng:
        phi0 = np.array([x[0, 0] for x in k._svmt_run(eng, wrap(X))])
        full = np.outer(phi0, phi0)
        Ks, _, _ = eng.gram(len(X), row_range=(3, 40))
        assert _eq(Ks, full[3:40])
        dev = torch.empty((len(X), len(X)), dtype=torch.float64, device="cuda")
        eng.gram(len(X), device_ptr=dev.data_ptr(), ld=len(X))
        torch.cuda.synchronize()
        assert _eq(dev.cpu().numpy(), full)
        phiy = np.array([y[0, 0] for y in k._svmt_run(eng, wrap(Y), fit_phi0=phi0)])
        Kt, xd, yd = eng.gram(len(X) + len(Y), n_fit=len(X), row_range=(1, 5))
        assert _eq(Kt, np.outer(phiy, phi0)[1:5])
        assert _eq(xd, phi0 * phi0) and _eq(yd, phiy * phiy)
    # reruns give the same result and pickling keeps the fitted state
    k2 = SvmTheta(random_state=5, subsets_size_range=(6, 8))
    a = k2.fit_transform(wrap(X))
    b = SvmTheta(random_state=5, subsets_size_range=(6, 8)).fit_transform(wrap(X))
    assert _eq(a, b)
    k3 = pickle.loads(pickle.dumps(k2))
    assert _eq(k3.transform(wrap(Y)), k2.transform(wrap(Y)))


def test_bad_index_is_an_error():
    with _lib.engine() as eng:
        eng.svmt_solve([3, 4], np.zeros((7, 4), np.uint32))
        counts = np.array([[1], [1]], dtype=np.int32)  # one sample of size 2 per graph
        with pytest.raises(_lib.GrakelB200Error, match="not a vertex of its graph"):
            eng.svmt_phi(2, counts, np.array([0, 3, 1, 2], dtype=np.uint8))
        phi, _, _ = eng.svmt_phi(2, counts, np.array([0, 1, 2, 3], dtype=np.uint8))
        assert phi.shape == (2, 1)


def test_non_converging_solve_is_an_error():
    """A directed graph on which libsvm cycles (the reference never returns): 10^7 iterations, then an error."""
    A = svmt_cases._rand_set(4, 20, 3, 11, 0.4, directed=True)[10]
    k = SvmTheta(random_state=0)
    t0 = time.perf_counter()
    with pytest.raises(_lib.GrakelB200Error, match="did not converge"):
        k.fit_transform([[A]])
    print("non-converging solve: %d vertices, %.1f s to the error" % (A.shape[0], time.perf_counter() - t0))


def test_cap_128():
    rs = np.random.RandomState(2)
    A = np.triu((rs.rand(128, 128) < 0.1).astype(float), 1)
    A = A + A.T
    k = SvmTheta(random_state=0, subsets_size_range=(120, 128), n_samples=3)
    k._keep_details = True
    K = k.fit_transform([[A]])
    o = oracle.SvmThetaOracle(random_state=0, subsets_size_range=(120, 128), n_samples=3)
    assert _eq(K, o.fit_transform([A]))
    _, alphas, iters = oracle.theta_alphas(A)
    assert _eq(k.details_["alpha"], alphas) and k.details_["iters"][0] == iters
    B = np.zeros((129, 129))
    with pytest.raises(NotImplementedError):
        SvmTheta().fit_transform([[B]])
