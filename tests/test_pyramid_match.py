"""PyramidMatch without a GPU: the host embedding stage under a seeded `eigs` against the reference's goldens bit for
bit, the NumPy restatement against every golden K, the reference's errors, pickling, GraphKernel / WeisfeilerLehman
dispatch and the C-ABI declarations."""
import os
import pickle
import re
import sys
import warnings

import numpy as np
import pytest
from scipy.sparse.linalg import eigs as scipy_eigs

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import make_golden_pyramid_match as mg  # noqa: E402
import pm_oracle  # noqa: E402
from grakel_b200 import GraphKernel, PyramidMatch, WeisfeilerLehman, _lib, kernels  # noqa: E402
from grakel_b200.packing import adjacency_and_labels  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "pyramid_match.npz"))
GEN = mg.unpack_generated(GOLDEN)
INPUTS = mg.inputs(GEN)
WL_INPUTS = mg.wl_inputs(GEN)
CASES = [(name, spec) for name, (_, _, specs) in INPUTS.items() for spec in specs
         if mg.case_key(name, spec) + "__K_fit" in GOLDEN]
ERR_CASES = [(name, spec) for name, (_, _, specs) in INPUTS.items() for spec in specs
             if mg.case_key(name, spec) + "__err" in GOLDEN]
WL_CASES = [(name, spec) for name, (_, _, specs) in WL_INPUTS.items() for spec in specs]


def golden_calls(key):
    return pm_oracle.split_calls(GOLDEN[key + "__U"], GOLDEN[key + "__shapes"])


def raw_labels(G):
    return [adjacency_and_labels(x[0], x[1])[1] for x in G]


@pytest.fixture
def seeded(monkeypatch):
    """kernels.eigs with one seeded default_rng, as the golden generator wraps the reference's."""
    def use(seed):
        rng = np.random.default_rng(seed)
        monkeypatch.setattr(kernels, "eigs", lambda *a, **k: scipy_eigs(*a, rng=rng, **k))
    return use


def _port_calls(data):
    """The port's embeddings as per-call arrays, set-major (= the reference's call order)."""
    gp = np.concatenate([[0], np.cumsum(data.sizes)])
    return [data.U[s, gp[g]:gp[g + 1], :data.n_cols[s, g]] for s in range(data.U.shape[0]) for g in range(len(data))]


def _same_calls(port, gold):
    assert len(port) == len(gold)
    for a, b in zip(port, gold):
        assert a.shape == b.shape and np.array_equal(a, b)


@pytest.mark.parametrize("name,spec", CASES, ids=lambda x: str(x))
def test_host_embeddings_equal_goldens(name, spec, seeded):
    X, Y, _ = INPUTS[name]
    wl, L, d, norm, seed = spec
    seeded(seed)
    est = PyramidMatch(with_labels=wl, L=L, d=d, normalize=norm)
    est.fit(X)
    est._method_calling = 3
    Yd = est.parse_input(Y)
    _same_calls(_port_calls(est.X) + _port_calls(Yd), golden_calls(mg.case_key(name, spec)))


@pytest.mark.parametrize("name,spec", ERR_CASES, ids=lambda x: str(x))
def test_host_stage_fails_as_the_reference(name, spec, seeded):
    """Where the reference's run raised (ARPACK on a graph of more than d + 1 vertices without an edge), the port's
    host stage raises the same error type."""
    X, Y, _ = INPUTS[name]
    wl, L, d, norm, seed = spec
    seeded(seed)
    est = PyramidMatch(with_labels=wl, L=L, d=d, normalize=norm)
    with pytest.raises(Exception) as e:
        est.fit(X)
        est._method_calling = 3
        est.parse_input(Y)
    assert type(e.value).__name__ == str(GOLDEN[mg.case_key(name, spec) + "__err"])


@pytest.fixture
def recorded(monkeypatch):
    """Every |U| the port's host stage makes, in call order."""
    calls = []
    f = kernels.pm_embedding
    monkeypatch.setattr(kernels, "pm_embedding", lambda A, d: calls.append(f(A, d)) or calls[-1])
    return calls


@pytest.mark.parametrize("name,spec", WL_CASES, ids=lambda x: str(x))
def test_wl_host_embeddings_equal_goldens(name, spec, seeded, recorded):
    X, Y, _ = WL_INPUTS[name]
    h, wl, L, d, norm, seed = spec
    seeded(seed)
    est = WeisfeilerLehman(n_iter=h, base_graph_kernel=(PyramidMatch, {"with_labels": wl, "L": L, "d": d}))
    est.fit(X)
    est._method_calling = 3
    est.parse_input(Y)
    _same_calls(recorded, golden_calls(mg.case_key(name, spec)))


def _shuffled(G, seed):
    """The same graphs with every labels dictionary in another key order."""
    rs = np.random.RandomState(seed)
    out = []
    for x in G:
        keys = list(x[1])
        rs.shuffle(keys)
        out.append([x[0], {k: x[1][k] for k in keys}])
    return out


@pytest.mark.parametrize("name", sorted(WL_INPUTS))
def test_wl_embedding_rows_follow_their_vertices(name, seeded):
    """The packed WL block lists a graph's vertices in its labels dictionary's order: every embedding row sits at its
    own vertex's packed position, whatever that order, and a labelled vertex outside the edge dictionary has none."""
    from grakel_b200.packing import adjacency_and_order
    X = WL_INPUTS[name][0]
    for G in (X, _shuffled(X, 1), [[x[0], dict(reversed(list(x[1].items())))] for x in X]):
        seeded(0)
        est = WeisfeilerLehman(n_iter=1, base_graph_kernel=(PyramidMatch, {"d": 4})).fit(G)
        pm = est.X.pm
        gp = np.asarray(est.X.block.graph_ptr)
        seeded(0)
        ref = kernels.pm_embed_sets([adjacency_and_order(x[0])[0] for x in G], 4, 2)[0]
        base = 0
        for g, x in enumerate(G):
            A, order = adjacency_and_order(x[0])
            loc = {k: i for i, k in enumerate(order)}
            for i, k in enumerate(x[1]):
                v = gp[g] + i
                if k in loc:
                    assert (pm.skip is None or not pm.skip[v]) and np.array_equal(pm.U[:, v], ref[:, base + loc[k]])
                else:
                    assert pm.skip[v] and not pm.U[:, v].any()
            base += A.shape[0]


@pytest.mark.parametrize("name,spec", CASES, ids=lambda x: str(x))
def test_restatement_reproduces_goldens(name, spec):
    X, Y, _ = INPUTS[name]
    wl, L, d, norm, _ = spec
    key = mg.case_key(name, spec)
    us = golden_calls(key)
    lx, ly = (raw_labels(X), raw_labels(Y)) if wl else (None, None)
    K, Kt = pm_oracle.kernel(us[:len(X)], L, d, lx, us[len(X):], ly, normalize=norm)
    assert np.array_equal(K, GOLDEN[key + "__K_fit"], equal_nan=True)
    assert np.array_equal(Kt, GOLDEN[key + "__K_tr"], equal_nan=True)


def test_quirk_of_the_combine():
    """Both statements of the combine sit inside the level loop: at L = 2 a self similarity is 1.5 x the mass."""
    u = [np.array([[0.1, 0.7], [0.2, 0.9], [0.6, 0.3]])]
    K, _ = pm_oracle.kernel(u, 2, 2)
    assert K[0, 0] == 1.5 * 6
    assert pm_oracle.kernel(u, 0, 2)[0][0, 0] == 0


@pytest.mark.parametrize("name", sorted(mg.error_cases()))
def test_errors_of_the_reference(name):
    kw, X = mg.error_cases()[name]
    want = str(GOLDEN["err__" + name])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception) as e:
            PyramidMatch(**kw).fit_transform(X)
    assert type(e.value).__name__ == want


def test_validation_messages():
    for kw, msg in (({"with_labels": 1}, "with labels must be a boolean variable"),
                    ({"L": -1}, "L: the number of levels must be an integer bigger equal to 0"),
                    ({"d": 0}, "d: hypercube dimension must be an integer bigger than 1")):
        with pytest.raises(TypeError, match=re.escape(msg)):
            PyramidMatch(**kw).initialize()
    with pytest.raises(TypeError, match="L: the number"):
        WeisfeilerLehman(base_graph_kernel=(PyramidMatch, {"L": 2.0})).initialize()


def test_fitted_state_pickles(seeded):
    X, Y, _ = INPUTS["gen"]
    seeded(3)
    est = PyramidMatch(L=3, d=4).fit(X)
    est2 = pickle.loads(pickle.dumps(est))
    assert np.array_equal(est2.X.U, est.X.U) and np.array_equal(est2.X.n_cols, est.X.n_cols)
    assert est2._labels == est._labels and est2._num_labels == est._num_labels
    wl = WeisfeilerLehman(n_iter=2, base_graph_kernel=PyramidMatch).fit(X)
    wl2 = pickle.loads(pickle.dumps(wl))
    assert np.array_equal(wl2.X.pm.U, wl.X.pm.U)


def test_transform_does_not_embed_fitted_graphs_again(seeded, monkeypatch):
    X, Y, _ = INPUTS["gen"]
    seeded(3)
    est = PyramidMatch(L=3, d=4).fit(X)
    n = []
    monkeypatch.setattr(kernels, "pm_embedding", lambda A, d, _f=kernels.pm_embedding: n.append(1) or _f(A, d))
    est._method_calling = 3
    est.parse_input(Y)
    assert len(n) == len(Y)


def test_dispatch():
    gk = GraphKernel(kernel={"name": "PM", "L": 3, "d": 4, "with_labels": False})
    gk.initialize()
    assert type(gk.kernel_) is PyramidMatch and gk.kernel_.L == 3 and gk.kernel_.with_labels is False
    gk = GraphKernel(kernel="pyramid_match")
    gk.initialize()
    assert type(gk.kernel_) is PyramidMatch
    gk = GraphKernel(kernel=["WL", "PM"])
    gk.initialize()
    assert type(gk.kernel_) is WeisfeilerLehman and gk.kernel_.base_graph_kernel[0] is PyramidMatch
    gk.kernel_.initialize()
    WeisfeilerLehman(base_graph_kernel=(PyramidMatch, {"with_labels": False})).initialize()
    with pytest.raises(NotImplementedError):
        GraphKernel(kernel=["CORE", "PM"]).fit_transform(INPUTS["gen"][0])


def test_c_abi_declared():
    assert {"gk_pm_features", "gk_pm_cells"} <= set(_lib.exported_symbols())
    header = open(os.path.join(HERE, "..", "include", "grakel_b200.h")).read()
    assert re.search(r"int gk_pm_features\(gk_handle\* h, int32_t n_iter, int32_t L, int32_t d, const double\* U,\s*"
                     r"const int32_t\* n_cols,\s*const uint8_t\* skip, int32_t n_sets, int32_t flags, gk_stats\* stats\);",
                     header)
    assert "int gk_pm_cells(gk_handle* h, int32_t set, int32_t level, int64_t* out);" in header
    assert "#define GK_PM_LABELS 1" in header and "#define GK_PM_WL_LABELS 2" in header
    assert (_lib.GK_PM_LABELS, _lib.GK_PM_WL_LABELS) == (1, 2)


def test_graph_objects_and_blocks_are_accepted(seeded, monkeypatch):
    """grakel_b200.Graph elements (PyramidMatch and WeisfeilerLehman over it) and a read_tu block (PyramidMatch): the
    host stage makes the embeddings of the equivalent list input."""
    from grakel_b200 import Graph
    from grakel_b200.packing import Block
    X = INPUTS["mutag"][0][:10]
    seeded(5)
    a = PyramidMatch(d=4).fit(X).X
    seeded(5)
    b = PyramidMatch(d=4).fit([Graph(x[0], x[1]) for x in X]).X
    assert np.array_equal(a.U, b.U) and a.labels == b.labels
    seeded(5)
    w1 = WeisfeilerLehman(n_iter=1, base_graph_kernel=(PyramidMatch, {"d": 4})).fit(X).X.pm
    seeded(5)
    w2 = WeisfeilerLehman(n_iter=1, base_graph_kernel=(PyramidMatch, {"d": 4})).fit([Graph(x[0], x[1]) for x in X]).X.pm
    assert np.array_equal(w1.U, w2.U)
    # a block of edge-vertex graphs with unit weights: the adjacency of the same edge sets
    els = [adjacency_and_labels(x[0], x[1]) for x in X]
    gp = np.concatenate([[0], np.cumsum([A.shape[0] for A, _ in els])])
    rows = [np.nonzero(A[i])[0] + gp[g] for g, (A, _) in enumerate(els) for i in range(A.shape[0])]
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows])])
    blk = Block(gp, rp, np.concatenate(rows), None, [l for _, L in els for l in L])
    blk.mode = "sp"
    seeded(5)
    c = PyramidMatch(d=4).fit(blk).X
    assert np.array_equal(a.U, c.U) and a.labels == c.labels
