"""Host-side tests of Propagation / PropagationAttr: the draws, the label enumeration and the transition matrices
against the real reference's goldens, the stacked normalisation, validation in the reference's order, set_params,
pickling, GraphKernel dispatch and the C-ABI symbols.  No GPU needed."""
import json
import os
import pickle
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_golden_propagation import as_input, min_metric, raw_input, unflat  # noqa: E402
from grakel_b200 import GraphKernel, Propagation, PropagationAttr, _lib  # noqa: E402
from grakel_b200.kernels import row_normalized  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "propagation.npz"))
ALL = sorted({k.split("/")[0] for k in GOLD.files})
CASES = [c for c in ALL if not c.startswith("error_")]


def case(name):
    meta = json.loads(str(GOLD[name + "/meta"]))
    if meta["extra"].get("raw"):
        return meta, raw_input(meta["raw_X"]), (raw_input(meta["raw_Y"]) if meta["raw_Y"] else None)
    get = lambda tag: unflat(*(GOLD[name + "/" + tag + "_" + k] for k in ("sizes", "A", "hasT", "T", "L")))
    X = as_input(get("X"), meta["extra"])
    Y = as_input(get("Y"), meta["extra"]) if name + "/Y_sizes" in GOLD else None
    return meta, X, Y


def estimator(meta):
    p = dict(meta["params"])
    if meta["extra"].get("metric") == "min":
        p["metric"] = min_metric
    if p.get("random_state") == "RandomState(12)":
        p["random_state"] = np.random.RandomState(12)
    if meta["cls"] == "GK":
        return GraphKernel(**p)
    return (Propagation if meta["cls"] == "PR" else PropagationAttr)(**p)


@pytest.mark.parametrize("name", CASES)
def test_draws_and_enumeration_equal_reference(name):
    meta, X, _ = case(name)
    est = estimator(meta)
    est.fit(X)
    if meta["extra"].get("second_fit"):
        est.fit(X)
    kern = est.kernel_ if meta["cls"] == "GK" else est
    assert np.array_equal(np.stack(kern._u), GOLD[name + "/u"])
    assert np.array_equal(np.stack([np.atleast_1d(b) for b in kern._b]), GOLD[name + "/b"])
    if not kern.attr_:
        assert list(kern._enum_labels) == GOLD[name + "/enum"].tolist()
        assert list(kern._enum_labels.values()) == GOLD[name + "/enum_ids"].tolist()
        assert kern._parent_labels == set(GOLD[name + "/enum"].tolist())
    else:
        assert kern._dim == GOLD[name + "/u"].shape[1]


def test_stacked_normalisation_equals_per_matrix_calls():
    from sklearn.preprocessing import normalize
    rs = np.random.RandomState(0)
    mats = []
    for k in range(60):
        n = [1, 3, 3, 5, 8][k % 5]
        A = rs.rand(n, n) * (rs.rand(n, n) < 0.5) * rs.choice([1.0, -1.0, 1e-7, 3e5], size=(n, n))
        if n > 2:
            A[1, :] = 0
        mats.append(A if k % 7 else (A != 0).astype(np.int64))
    mats.append(rs.rand(4, 4).astype(np.float32))
    for got, A in zip(row_normalized(mats), mats):
        want = normalize(A, axis=1, norm="l1")
        assert got.dtype == want.dtype and got.tobytes() == want.tobytes()


def test_transition_matrices_are_the_references():
    meta, X, _ = case("user_transition")
    from sklearn.preprocessing import normalize
    k = Propagation(t_max=3).fit(X)
    for T, x in zip(k.X.T, X):
        assert np.array_equal(T, normalize(x[3] if len(x) == 4 else x[0], axis=1, norm="l1"))


A3 = np.array([[0., 1., 0.], [1., 0., 1.], [0., 1., 0.]])


@pytest.mark.parametrize("params,exc,msg", [
    (dict(M="L1"), TypeError, 'Metric type must be a str, one of "H", "TV"'),
    (dict(M=3, t_max=0), TypeError, 'Metric type must be a str, one of "H", "TV"'),
    (dict(t_max=0, w=0), TypeError, "The number of iterations must be a positive integer."),
    (dict(t_max=2.0), TypeError, "The number of iterations must be a positive integer."),
    (dict(t_max=65), NotImplementedError, "at most t_max = 64"),
    (dict(w=0), NotImplementedError, "w = 0"),
    (dict(n_jobs="x", M="bad"), ValueError, "n_jobs parameter must be an int"),
])
def test_validation_in_reference_order(params, exc, msg):
    with pytest.raises(exc, match=msg.replace("(", r"\(").replace(")", r"\)")):
        Propagation(**params).fit([[A3, {0: 1, 1: 2, 2: 1}]])


def test_attr_validation():
    with pytest.raises(TypeError, match='"L1", "L2"'):
        PropagationAttr(M="TV").fit([[A3, {0: [1.], 1: [2.], 2: [3.]}]])
    with pytest.raises(ValueError, match="Attribute dimensions should be the same, for all graphs"):
        PropagationAttr().fit([])
    with pytest.raises(ValueError, match="Attribute dimensions should be the same"):
        PropagationAttr().fit([[A3, {0: [1.], 1: [2.], 2: [3.]}], [A3, {0: [1., 2], 1: [2., 2], 2: [3., 2]}]])
    k = PropagationAttr().fit([[A3, {0: [1.], 1: [2.], 2: [3.]}]])
    k._method_calling = 3
    with pytest.raises(ValueError, match="same dimension as in fit"):
        k.parse_input([[A3, {0: [1., 0], 1: [2., 0], 2: [3., 0]}]])
    with pytest.raises(NotImplementedError, match="dtype"):
        PropagationAttr().fit([[A3, {0: [True], 1: [False], 2: [True]}]])


def test_quirks_kept():
    # w < 0 passes, a non-callable metric is never rejected at initialize
    Propagation(w=-0.5, metric=3).fit([[A3, {0: 1, 1: 2, 2: 1}]])
    with pytest.raises(ValueError, match="input must be an iterable"):
        Propagation().fit(3)
    with pytest.raises(ValueError, match="Each element of X must be either a Graph"):
        Propagation().fit([[A3]])
    with pytest.raises(ValueError, match="Parsed input is empty"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            Propagation().fit([[]])
    with pytest.raises(TypeError, match="must be a square matrix"):
        Propagation().fit([[A3, {0: 1, 1: 2, 2: 1}, {}, np.zeros((3, 2))]])
    with pytest.raises(TypeError, match="same dimension as the number of vertices"):
        Propagation().fit([[A3, {0: 1, 1: 2, 2: 1}, {}, np.zeros((2, 2))]])
    with pytest.raises(TypeError, match="labels should be hashable"):
        Propagation().fit([[A3, {0: [1], 1: [2], 2: [1]}]])
    import scipy.sparse as sp
    with pytest.raises(ValueError, match="setting an array element with a sequence"):
        Propagation(t_max=2).fit([[A3, {0: 1, 1: 2, 2: 1}, {}, sp.csr_matrix(A3)]])
    Propagation(t_max=1).fit([[A3, {0: 1, 1: 2, 2: 1}, {}, sp.csr_matrix(A3)]])


def test_set_params_reinitialises():
    k = Propagation(random_state=0, t_max=3).fit([[A3, {0: 1, 1: 2, 2: 1}]])
    assert len(k._u) == 3 and not k.take_sqrt_
    k.set_params(t_max=2)
    k.fit([[A3, {0: 1, 1: 2, 2: 1}]])
    assert len(k._u) == 2
    # the reference validates M under the "metric" flag: changing M alone keeps the fitted choice
    k.set_params(M="H")
    k.fit([[A3, {0: 1, 1: 2, 2: 1}]])
    assert not k.take_sqrt_
    k.set_params(metric=k.metric)
    k.fit([[A3, {0: 1, 1: 2, 2: 1}]])
    assert k.take_sqrt_
    k.set_params(t_max=0)
    with pytest.raises(TypeError):
        k.fit([[A3, {0: 1, 1: 2, 2: 1}]])


def test_fitted_estimators_pickle():
    meta, X, _ = case("generated_new_label")
    k = estimator(meta).fit(X)
    k2 = pickle.loads(pickle.dumps(k))
    assert all(np.array_equal(a, b) for a, b in zip(k._u, k2._u)) and k._b == k2._b
    assert k2._enum_labels == k._enum_labels and k2.random_state_.randn() == k.random_state_.randn()
    ka = PropagationAttr(random_state=0).fit([[A3, {0: [1.], 1: [2.], 2: [3.]}]])
    assert pickle.loads(pickle.dumps(ka))._dim == 1


def test_graph_kernel_dispatch_and_random_state():
    gk = GraphKernel(kernel="PR", random_state=5)
    gk.initialize()
    assert type(gk.kernel_) is Propagation and gk.kernel_.random_state is gk.random_state_
    gk = GraphKernel(kernel={"name": "propagation", "with_attributes": True, "random_state": 3}, random_state=5)
    gk.initialize()
    assert type(gk.kernel_) is PropagationAttr and gk.kernel_.random_state == 3
    gk = GraphKernel(kernel="PR")
    gk.initialize()
    assert gk.kernel_.random_state is None
    # WL and CORE over PR stay outside the device hot path
    with pytest.raises(NotImplementedError):
        GraphKernel(kernel=["WL", "PR"]).fit([[A3, {0: 1, 1: 2, 2: 1}]])


def test_c_abi_symbols():
    assert {"gk_pk_features", "gk_pk_hashes"} <= set(_lib.exported_symbols())
    names = [n for n, _ in _lib.GkStats._fields_]
    assert names[-2:] == ["ms_propagate", "pk_near_edge"]
    header = open(os.path.join(HERE, "..", "include", "grakel_b200.h")).read()
    assert "int gk_pk_features(" in header and "int gk_pk_hashes(" in header


# ---- the NumPy restatement against the reference's goldens
import pk_oracle as O  # noqa: E402


def restated(kern, data, fit_sizes=None, transform=False):
    """(levels, split) of the restatement for parsed data `data` of a fitted estimator."""
    if kern.attr_:
        return O.levels(data.T, data.sizes, data.P, kern._u, kern._b, kern.w, attr=True), False
    P = np.zeros((len(data.ids), data.dim))
    P[np.arange(len(data.ids)), data.ids] = 1.0
    split = transform and data.u_full is not None
    us = data.u_full if split else kern._u
    return O.levels(data.T, data.sizes, P, us, kern._b, kern.w, sqrt=kern.take_sqrt_,
                    dim_orig=len(kern._enum_labels) if split else None, labels=data.ids), split


def _normalised(K, dy, dx):
    with np.errstate(invalid="ignore", divide="ignore"):
        return K / np.sqrt(np.outer(dy, dx))


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference(name):
    meta, X, Y = case(name)
    est = estimator(meta)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        est.fit(X)
        if meta["extra"].get("second_fit"):
            est.fit(X)
    kern = est.kernel_ if meta["cls"] == "GK" else est
    lx, _ = restated(kern, kern.X)
    for t, (b, priv) in enumerate(lx):
        assert np.array_equal(b.reshape(GOLD[name + "/call%d" % t].shape), GOLD[name + "/call%d" % t]), t
    cx = O.counts(lx, kern.X.sizes)
    K, dx = O.gram(cx), O.diag(cx)
    if meta["params"].get("normalize"):
        K = _normalised(K, dx, dx)
    if "metric" not in meta["extra"]:
        assert np.array_equal(K, GOLD[name + "/K"])
    if Y is None:
        return
    kern._method_calling = 3
    Yd = kern.parse_input(Y)
    ly, split = restated(kern, Yd, transform=True)
    calls = [GOLD[name + "/call%d" % i] for i in range(meta["n_fit_calls"], meta["n_calls"])]
    for t, (b, priv) in enumerate(ly):
        if split:
            assert np.array_equal(b[~priv], calls[2 * t]) and np.array_equal(b[priv], calls[2 * t + 1]), t
        else:
            assert np.array_equal(b.reshape(calls[t].shape), calls[t]), t
    cy = O.counts(ly, Yd.sizes, split)
    Kt = O.gram(cx, cy)
    if meta["params"].get("normalize"):
        Kt = _normalised(Kt, O.diag(cy), dx)
    if "metric" not in meta["extra"]:
        assert np.array_equal(Kt, GOLD[name + "/Kt"])


def test_fortran_ordered_transition_normalises_like_the_reference():
    from sklearn.preprocessing import normalize
    rs = np.random.RandomState(3)
    mats = [np.asfortranarray(rs.rand(12, 12) * rs.choice([1e-9, 1.0, 7e5], size=(12, 12))) for _ in range(4)]
    mats += [np.ascontiguousarray(m) for m in mats]
    for got, A in zip(row_normalized(mats), mats):
        assert got.tobytes() == normalize(A, axis=1, norm="l1").tobytes()


def test_sparse_transition_error_is_the_references():
    meta, X, _ = case("error_sparse_transition")
    with pytest.raises(ValueError) as e:
        estimator(meta).fit_transform(X)
    assert [type(e.value).__name__, str(e.value)] == meta["err"]
    # raised after the fit's draws, as the reference raises it at its first propagation step
    k = estimator(meta)
    with pytest.raises(ValueError):
        k.fit(X)
    ref = np.random.RandomState(meta["params"]["random_state"])
    for _ in range(meta["params"]["t_max"]):
        ref.randn(len(k._enum_labels)); ref.randn(len(k._enum_labels)); ref.rand()
    assert k.random_state_.randn() == ref.randn()


def test_validation_interleaves_normalisation_and_labels():
    # element 0's T cannot be normalised (NaN entries), element 1's labels are unhashable: the reference
    # normalises element 0 before it looks at element 1's labels
    bad_T = np.full((3, 3), np.nan)
    X = [[A3, {0: 1, 1: 2, 2: 1}, {}, bad_T], [A3, {0: [1], 1: [2], 2: [1]}]]
    from sklearn.preprocessing import normalize
    with pytest.raises(Exception) as ref:
        normalize(bad_T, axis=1, norm="l1")
    with pytest.raises(type(ref.value), match="NaN"):
        Propagation().fit(X)
