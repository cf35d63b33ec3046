"""Propagation / PropagationAttr on the H100 against the real reference's goldens: every level's bins (the new-label
split included), K of fit_transform and transform bit for bit, the Gram variants, determinism."""
import functools
import os
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))

from test_propagation import CASES, GOLD, case, estimator, restated  # noqa: E402
import pk_oracle as O  # noqa: E402
from grakel_b200 import _lib  # noqa: E402

pytestmark = pytest.mark.gpu


def _bins_of(kern, X, Y):
    with _lib.engine() as eng:
        st, V, _, _ = kern._pk_features(eng, X, Y)
        width = kern._dim if kern.attr_ else 1
        return st, [eng.pk_hashes(t, V, width) for t in range(kern.t_max)]


def _same(dev, ref):
    dev = dev.reshape(ref.shape) if ref.ndim == 2 else dev.ravel()
    return dev.shape == ref.shape and np.array_equal(dev, ref)


@pytest.mark.parametrize("name", CASES)
def test_golden_case(name):
    meta, X, Y = case(name)
    est = estimator(meta)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        K = est.fit_transform(X)
        if meta["extra"].get("second_fit"):
            K = est.fit_transform(X)
        kern = est.kernel_ if meta["cls"] == "GK" else est
        assert np.array_equal(K, GOLD[name + "/K"])
        # fit bins, level by level
        st, bins = _bins_of(kern, kern.X, None)
        for t in range(kern.t_max):
            assert _same(bins[t][0], GOLD[name + "/call%d" % t]), t
            assert not bins[t][1].any()
        if Y is None:
            return
        # transform: the reference's draws continue the stream, so the estimator's own transform comes first
        seen = {}
        kern._pk_features = functools.partial(_capture, kern, seen)
        Kt = est.transform(Y)
        assert np.array_equal(Kt, GOLD[name + "/Kt"])
    bins, Vx = seen["bins"], int(np.sum(kern.X.sizes))
    calls = [GOLD[name + "/call%d" % i] for i in range(meta["n_fit_calls"], meta["n_calls"])]
    split = len(calls) == 2 * kern.t_max
    for t in range(kern.t_max):
        b, priv = bins[t][0][Vx:], bins[t][1][Vx:]
        if not split:
            assert _same(b, calls[t]) and not priv.any(), t
        else:
            assert _same(b[~priv], calls[2 * t]), t
            assert _same(b[priv], calls[2 * t + 1]), t


def _capture(kern, seen, eng, X, Y):
    st, V, n, n_fit = type(kern)._pk_features(kern, eng, X, Y)
    width = kern._dim if kern.attr_ else 1
    seen["bins"] = [eng.pk_hashes(t, V, width) for t in range(kern.t_max)]
    return st, V, n, n_fit


def _engine_run(kern, Y=None, **gram_kw):
    with _lib.engine() as eng:
        st, _, n, n_fit = kern._pk_features(eng, kern.X, Y)
        K, xd, yd = eng.gram(n, n_fit=n_fit, stats=st, **gram_kw)
    return K, st


@pytest.mark.parametrize("name,transform", [("mutag_tv", False), ("mutag_tv", True), ("attr_generated_l1", True),
                                            ("directed_signed", False)])
def test_gram_variants_equal_default(name, transform, monkeypatch):
    meta, X, Y = case(name)
    kern = estimator(meta)
    kern.fit(X)
    Yd = None
    if transform:
        kern._method_calling = 3
        Yd = kern.parse_input(Y)
    K, st = _engine_run(kern, Yd)
    assert st.gram_path in (1, 2, 3)
    for T in ("1", "4096"):
        monkeypatch.setenv("GRAKEL_B200_FORCE_T", T)
        assert np.array_equal(_engine_run(kern, Yd)[0], K), T
    monkeypatch.delenv("GRAKEL_B200_FORCE_T")
    assert np.array_equal(_engine_run(kern, Yd, simt=True)[0], K)
    rows = K.shape[0]
    a, b = rows // 3, rows // 3 + max(1, rows // 4)
    assert np.array_equal(_engine_run(kern, Yd, row_range=(a, b))[0], K[a:b])
    assert np.array_equal(_engine_run(kern, Yd, dtype=np.float32)[0], K.astype(np.float32))
    import torch
    out = torch.full((rows, K.shape[1] + 3), float("nan"), dtype=torch.float64, device="cuda")
    _engine_run(kern, Yd, device_ptr=out.data_ptr(), ld=K.shape[1] + 3)
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.array_equal(o[:, :K.shape[1]], K) and np.all(np.isnan(o[:, K.shape[1]:]))
    with pytest.raises(NotImplementedError, match="GK_DIST"):
        _engine_run(kern, Yd, dist=True, row_range=(0, rows))


def test_two_runs_bit_identical():
    import bench
    X = bench.gen_list(600, 40, 0)
    from grakel_b200 import Propagation
    k1 = Propagation(random_state=0)
    K1 = k1.fit_transform(X)
    _, b1 = _bins_of(k1, k1.X, None)
    K2 = k1.fit_transform(X)  # new draws: a different K, but the same K for the same draws below
    k3 = Propagation(random_state=0)
    K3 = k3.fit_transform(X)
    _, b3 = _bins_of(k3, k3.X, None)
    assert np.array_equal(K1, K3) and not np.array_equal(K1, K2)
    assert all(np.array_equal(x[0], y[0]) for x, y in zip(b1, b3))
    assert k1.stats_.n_levels == 5 and k1.stats_.n_columns > 0


def test_nan_bins_raise_key_error():
    from grakel_b200 import Propagation
    A = np.array([[0., -1., 0.], [1., 0., 1.], [0., 1., 0.]])
    with pytest.raises(KeyError):
        Propagation(random_state=0, M="H", t_max=3).fit_transform([[A, {0: 1, 1: 2, 2: 1}]])


def test_read_tu_block_equals_list_input():
    """A read_tu(kernel="SP") block walks the nodes that occur in an edge, as the reference's edge dictionaries do."""
    import tempfile
    import make_golden_neighborhood_hash as mg
    from make_golden_tu import unpack
    from grakel_b200 import Propagation
    from grakel_b200.datasets import read_tu
    d = tempfile.mkdtemp()
    unpack("MUTAG", d)
    block = read_tu(d, "MUTAG", kernel="SP").data
    Kb = Propagation(random_state=1, t_max=3).fit_transform(block)
    Kl = Propagation(random_state=1, t_max=3).fit_transform(mg.mutag())
    assert np.array_equal(Kb, Kl)


@pytest.mark.parametrize("name", [c for c in CASES if GOLD[c + "/u"].ndim == 2])
def test_lazy_hd_is_the_references(name):
    meta, X, _ = case(name)
    est = estimator(meta)
    est.fit(X)
    if meta["extra"].get("second_fit"):
        est.fit(X)
    kern = est.kernel_ if meta["cls"] == "GK" else est
    for t, hd in enumerate(kern._hd):
        h = GOLD[name + "/call%d" % t]
        if kern.attr_:
            want = {j: i for i, j in enumerate({tuple(l) for l in h.tolist()})}
        else:
            want = dict((j, i) for i, j in enumerate(set(np.unique(h))))
        assert list(hd.items()) == list(want.items()), t


def test_nan_error_is_the_references():
    meta, X, _ = case("error_h_negative")
    with pytest.raises(KeyError) as e:
        estimator(meta).fit_transform(X)
    assert [type(e.value).__name__, str(e.value)] == meta["err"]


def test_near_edge_counts_exact_integers():
    # one graph, labels 0 1 0: level 0 hashes (u[l] + b) / w exactly
    gp, rp, ci = np.array([0, 3]), np.array([0, 1, 3, 4]), np.array([1, 0, 2, 1], dtype=np.int32)
    tv = np.array([1.0, 0.5, 0.5, 1.0])
    ids = np.array([0, 1, 0], dtype=np.int32)
    with _lib.engine() as eng:
        eng.pack(gp, rp, ci, ids, None, None)
        on = eng.pk_features(1, 0.5, np.array([[1.0, 2.0]]), np.array([0.0]), 2, 2, 1, tv)
        off = eng.pk_features(1, 1.0, np.array([[0.3, 0.1]]), np.array([0.25]), 2, 2, 1, tv)
        # after one step vertex 1 holds (1, 0): (1 * 0.5 + 0) / 0.5 = 1 exactly at level 1 as well
        two = eng.pk_features(2, 0.5, np.array([[1.0, 2.0], [0.5, 0.25]]), np.array([0.0, 0.0]), 2, 2, 1, tv)
    assert on.pk_near_edge == 3 and off.pk_near_edge == 0 and two.pk_near_edge >= 4


def test_scale_bins_and_gram_match_the_restatement():
    """bench.gen_list(10000, 40, 0), Propagation(t_max=5, w=0.01): device bins equal the restatement's except among
    the near-edge hashes, and K equals the restatement's where no hash is near an edge."""
    import bench
    import scipy.sparse as sp
    from grakel_b200 import Propagation
    X = bench.gen_list(10000, 40, 0)
    for M in ("TV", "H"):
        kern = Propagation(random_state=0, M=M).fit(X)
        st, dev = _bins_of(kern, kern.X, None)
        ref, _ = restated(kern, kern.X)
        mismatched = sum(int(np.sum(d[0].ravel() != r[0])) for d, r in zip(dev, ref))
        assert mismatched <= st.pk_near_edge, (M, mismatched, st.pk_near_edge)
        K = Propagation(random_state=0, M=M).fit_transform(X)
        if st.pk_near_edge:
            continue
        sizes = kern.X.sizes
        gidx = np.repeat(np.arange(len(sizes)), sizes)
        blocks = []
        for b, _ in ref:
            _, col = np.unique(b, return_inverse=True)
            blocks.append(sp.csr_matrix((np.ones(len(b)), (gidx, col.ravel())), shape=(len(sizes), col.max() + 1)))
        Phi = sp.hstack(blocks).tocsr()
        rows = np.random.RandomState(1).choice(len(sizes), 64, replace=False)
        Kr = (Phi[rows] @ Phi.T).toarray()
        assert np.array_equal(K[rows], Kr), M
