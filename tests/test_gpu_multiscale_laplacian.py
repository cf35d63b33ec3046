"""MultiscaleLaplacian on the device: the reference's goldens within 1e-9 relative, the sample blocks against the
oracle, symmetry, reruns, row blocks and device output, the caps at their edges, self-loops, and a bench-sized set."""
import warnings

import numpy as np
import pytest

import grakel_b200.kernels as kmod
from grakel_b200 import GraphKernel, MultiscaleLaplacian, _lib
from ml_cases import as_input, load, rel_err, replay_eig
from ml_oracle import MLOracle, flg_matrix

pytestmark = pytest.mark.gpu
META, CASES = load()
BAR = 1e-9


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("norm", [False, True])
def test_device_matches_golden(name, norm, monkeypatch):
    c = CASES[name]
    g = c["g"]
    monkeypatch.setattr(kmod, "ml_eig", replay_eig(g, c["levels"]))
    k = MultiscaleLaplacian(normalize=norm, **c["params"])
    K = k.fit_transform(as_input(c["X"]))
    sfx = "_norm" if norm else ""
    assert rel_err(K, g["K_fit" + sfx]) <= BAR
    assert rel_err(k.transform(as_input(c["Y"])), g["K_tr" + sfx]) <= BAR
    for l, vs in enumerate(k.samples_):
        assert [(a, b) for a, b in g["samples_%d" % l]] == vs


def test_reference_tests_workload():
    """The reference tests' workload with numpy's own eig: within the bar, exactly symmetric, diagonal 2^(-P'/2)."""
    c = CASES["reference_tests"]
    k = MultiscaleLaplacian(random_state=0)
    K = k.fit_transform(as_input(c["X"]))
    assert rel_err(K, c["g"]["K_fit"]) <= BAR
    assert np.array_equal(K, K.T)
    d = k.diagonal()
    assert np.array_equal(np.diagonal(K), d)
    Pw = k._data_level[3][1].shape[1]
    np.testing.assert_allclose(d, 2.0 ** (-Pw / 2), rtol=1e-9)
    Kt = k.transform(as_input(c["Y"]))
    assert rel_err(Kt, c["g"]["K_tr"]) <= BAR
    # a second fit on the same (normalising) estimator draws new samples, as the reference's does
    k2 = MultiscaleLaplacian(random_state=0, normalize=True)
    k2.fit_transform(as_input(c["X"]))
    assert rel_err(k2.fit_transform(as_input(c["X"])), c["g"]["K_refit"]) <= BAR
    gk = GraphKernel(kernel="ML", random_state=7)
    assert rel_err(gk.fit_transform(as_input(c["X"])), c["g"]["K_graphkernel"]) <= BAR


def test_sample_blocks_against_oracle():
    c = CASES["gamma_heta"]
    k = MultiscaleLaplacian(**c["params"])
    k.fit(as_input(c["X"]))
    o = MLOracle(**c["params"]).fit(c["X"])
    for l, (Cs, Q) in enumerate(o.levels, start=1):
        rec, Qd = k._data_level[l]
        P = int(round(np.sqrt(rec.shape[1] - 1)))
        recs = [(r[:-1].reshape(P, P), r[-1]) for r in rec]
        Kd = flg_matrix(recs, recs)
        assert rel_err(Kd, flg_matrix(Cs, Cs)) <= BAR


def test_reruns_rows_and_device_output():
    c = CASES["weighted_loops"]
    X = as_input(c["X"])
    K1 = MultiscaleLaplacian(**c["params"]).fit_transform(X)
    K2 = MultiscaleLaplacian(**c["params"]).fit_transform(X)
    assert np.array_equal(K1, K2) and np.array_equal(K1, K1.T)
    k = MultiscaleLaplacian(**c["params"])
    k.initialize()
    k._method_calling = 1
    els = k._elements(X)
    import torch
    with _lib.engine() as eng:
        k._ml_pipeline(eng, els)
        N = len(els)
        Kf, _, _ = eng.gram(N)
        Kr, _, _ = eng.gram(N, row_range=(2, 6))
        Kn, _, _ = eng.gram(N, normalize=True)
        dev = torch.zeros((N, N), dtype=torch.float64, device="cuda")
        eng.gram(N, device_ptr=dev.data_ptr())
        torch.cuda.synchronize()
    assert np.array_equal(Kf, K1)
    assert np.array_equal(Kr, Kf[2:6])
    assert np.array_equal(dev.cpu().numpy(), Kf)
    d = np.diagonal(Kf)
    np.testing.assert_allclose(Kn, Kf / np.sqrt(np.outer(d, d)), rtol=1e-15)


def _attr_set(seed, n_graphs, n, dim):
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n_graphs):
        A = np.triu((rs.rand(n, n) < 0.2).astype(float), 1)
        out.append((A + A.T, rs.rand(n, dim)))
    return out


def test_graph_size_cap():
    for n, ok in ((128, True), (129, False)):
        els = _attr_set(1, 3, n, 4)
        with _lib.engine() as eng:
            gp = np.array([0, n, 2 * n, 3 * n])
            rp = np.zeros(3 * n + 1, dtype=np.int32)
            eng.pack(gp, rp, np.zeros(0, dtype=np.int32), None, None, None)
            phi = np.concatenate([p for _, p in els])
            if ok:
                eng.ml_begin(2, 0.01, 0.01, phi)
            else:
                with pytest.raises(NotImplementedError):
                    eng.ml_begin(2, 0.01, 0.01, phi)


def test_width_cap():
    X = as_input(_attr_set(2, 6, 20, 40))
    K = MultiscaleLaplacian(random_state=0, L=1, P=32).fit_transform(X)
    assert np.array_equal(K, K.T)
    with pytest.raises(NotImplementedError):
        MultiscaleLaplacian(random_state=0, L=1, P=33).fit_transform(X)


def test_sample_cap():
    X = as_input(_attr_set(3, 41, 25, 3))
    K = MultiscaleLaplacian(random_state=0, L=1, P=3, n_samples=1024).fit_transform(X)
    assert np.all(np.isfinite(K))
    with pytest.raises(NotImplementedError):
        MultiscaleLaplacian(random_state=0, L=1, P=3, n_samples=1025).fit_transform(X)


def test_self_loop_multiplicity():
    """A self-loop lists its vertex twice in the level-1 neighbourhood: the device follows the oracle, and dropping
    the duplicate would change K."""
    els = _attr_set(4, 6, 9, 4)
    for i, (A, _) in enumerate(els):
        A[i % 9, i % 9] = 2.0
    o = MLOracle(random_state=3, L=2, P=4, n_samples=20)
    Ko = o.fit_transform(els)
    K = MultiscaleLaplacian(random_state=3, L=2, P=4, n_samples=20).fit_transform(as_input(els))
    assert rel_err(K, Ko) <= BAR


def test_bench_graphs_against_oracle():
    import bench
    X = bench.gen_list(200, 40, 0, attr=16, as_adj=True)
    els = [(np.asarray(A, dtype=float), np.array([list(L[i]) for i in range(len(L))])) for A, L in X]
    k = MultiscaleLaplacian(random_state=0, L=1)
    K = k.fit_transform(X[:150])
    Kt = k.transform(X[150:])
    o = MLOracle(random_state=0, L=1)
    assert rel_err(K, o.fit_transform(els[:150])) <= BAR
    assert rel_err(Kt, o.transform(els[150:])) <= BAR


def test_read_tu_block_with_attributes(tmp_path):
    """A datasets.read_tu block with node attributes: the attribute rows are the features."""
    from make_golden_tu import unpack
    from grakel_b200.datasets import read_tu
    unpack("Cuneiform", str(tmp_path))
    block = read_tu(str(tmp_path), "Cuneiform", kernel="SP", prefer_attr_nodes=True).data
    k = MultiscaleLaplacian(random_state=0, L=2, n_samples=30)
    K = k.fit_transform(block)
    els = k._elements(block)
    assert rel_err(K, MLOracle(random_state=0, L=2, n_samples=30).fit_transform(els)) <= BAR
