"""HadamardCode on the host: the NumPy restatement against the reference's goldens (every level vector and every K of
the VertexHistogram base, bit for bit), the popcount rows against scipy's Hadamard matrix, the enumeration replay, the
skip masks of every edge-dictionary spelling, the errors, GraphKernel dispatch, pickling and the C-ABI symbols."""
import os
import pickle
import sys
import warnings

import numpy as np
import pytest
import scipy.linalg

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import hc_oracle  # noqa: E402
from grakel_b200 import EdgeHistogram, GraphKernel, HadamardCode, ShortestPath, VertexHistogram, _lib, kernels  # noqa: E402
from make_golden_hadamard_code import ERRORS, GK_FORMS, inputs, same_width, spellings, unpack_generated  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "hadamard_code.npz"))
INPUTS = inputs(unpack_generated("gen8", GOLDEN))
CASES = sorted(INPUTS.items())
VH_CASES = [(n, s) for n, s in CASES if s.get("base", "VH") == "VH"]


def _warn_free(fn, *a):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a)


@pytest.mark.parametrize("name,spec", [c for c in VH_CASES if c[1].get("vec")], ids=lambda x: str(x))
def test_oracle_level_vectors(name, spec):
    enum = hc_oracle.enumerate_labels(x[1] for x in spec["X"])
    W = kernels.hc_width(len(enum))
    lv = hc_oracle.levels(spec["X"], spec["n_iter"], enum)
    for i in range(spec["n_iter"]):
        assert np.array_equal(hc_oracle.packed_rows(spec["X"], lv[i], W), GOLDEN["%s__vec%d" % (name, i)]), i


def test_wrap_case_wraps():
    """The complete graph on 65 vertices multiplies the common vector by 65 per level: level 11 passes 2^63."""
    v = GOLDEN["wrap__vec12"][:65]
    big = [np.abs(GOLDEN["wrap__vec%d" % i][:65].astype(object)).max() for i in range(13)]
    assert big[10] < 2 ** 63 and int(np.int64(65) ** 10) == big[10]
    assert not np.array_equal(GOLDEN["wrap__vec11"][:65].astype(object), np.full((65, 1), 65 ** 11, dtype=object))
    assert (v == v[0]).all()


@pytest.mark.parametrize("name,spec", VH_CASES, ids=lambda x: str(x))
def test_oracle_kernels(name, spec):
    if spec.get("normalize"):
        pytest.skip("normalised matrices are checked on the device")
    K, _ = _warn_free(hc_oracle.kernel, spec["X"], spec["n_iter"])
    assert np.array_equal(K, GOLDEN[name + "__K"])
    if spec.get("Y") is not None:
        enum = hc_oracle.enumerate_labels(x[1] for x in spec["X"])
        enum_all = hc_oracle.enumerate_labels((y[1] for y in spec["Y"]), enum)
        if kernels.hc_width(len(enum_all)) == kernels.hc_width(len(enum)):
            Kt, _ = _warn_free(hc_oracle.kernel, spec["X"], spec["n_iter"], spec["Y"])
            assert np.array_equal(Kt, GOLDEN[name + "__Kt"])
        else:  # the widths differ: nothing is shared
            assert not GOLDEN[name + "__Kt"].any()


def test_popcount_rows_are_scipy_hadamard():
    for W in (1, 2, 4, 8, 16, 64, 256, 1024):
        H = scipy.linalg.hadamard(W)
        assert H.dtype == np.int64
        for r in range(0, W, max(1, W // 64)):
            assert np.array_equal(hc_oracle.hadamard_row(r, W), H[r]), (W, r)


@pytest.mark.parametrize("name,spec", [c for c in CASES if c[1].get("enum")], ids=lambda x: str(x))
def test_enumeration_replay(name, spec):
    enum = kernels.hc_enumerate(x[1] for x in spec["X"])
    assert list(enum) == GOLDEN[name + "__enum_keys"].tolist()
    assert [enum[k] for k in enum] == GOLDEN[name + "__enum_ids"].tolist()


def test_width():
    assert [kernels.hc_width(n) for n in (1, 2, 3, 4, 5, 8, 9)] == [1, 2, 4, 4, 8, 8, 16]


def test_skip_masks_of_every_spelling():
    want = [
        [False, False, True],  # labelled vertex 5 is outside the edge dictionary
        [False, False],        # {0: {1: 1}}: the sink 1 is a key
        [False, False],        # {0: [1]}
        [False, False],        # {(0, 1): 1}
        [False, False, False],  # {u: {}} keeps u
        [False, False, True],  # {u: []} does not
        [False, False, False],
        [False, False],
        [False, False, False],
        [False, False, False, True],
    ]
    hc = HadamardCode(n_iter=2)
    hc.initialize()
    data, _ = hc._parse(spellings(), None)
    assert np.array_equal(data.skip, np.concatenate([np.array(w) for w in want]))
    for x, w in zip(spellings(), want):
        keys = kernels.hc_edge_keys(x[0])
        assert [k not in keys for k in x[1]] == w
    A = np.array([[0, 1], [0, 0]])
    assert kernels.hc_edge_keys(A) is None


def test_unlabelled_edge_key_raises_like_the_reference():
    X = [[{(0, 1): 1, (1, 2): 1}, {0: "a", 1: "b"}]] * 2
    hc = HadamardCode(n_iter=2)
    hc.initialize()
    with pytest.raises(KeyError):
        hc._parse(X, None)
    hc = HadamardCode(n_iter=1)
    hc.initialize()
    data, _ = hc._parse(X, None)  # level 0 only: the labels
    assert data.block.n_vertices == 4


@pytest.mark.parametrize("name", sorted(ERRORS))
def test_errors(name):
    kw = dict(ERRORS[name])
    X = kw.pop("X", same_width())
    if kw.get("base_graph_kernel") == ("VH_class", 5):
        kw["base_graph_kernel"] = (VertexHistogram, 5)
    err = str(GOLDEN[name + "__err"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises({"TypeError": TypeError, "ValueError": ValueError}[err]):
            HadamardCode(**kw).fit_transform(X)


def test_messages():
    with pytest.raises(TypeError, match="'n_iter' must be a positive integer"):
        HadamardCode(n_iter=0).initialize()
    with pytest.raises(ValueError, match="parsed input is empty"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            HadamardCode().fit([[]])
    with pytest.raises(NotImplementedError):
        HadamardCode(base_graph_kernel=kernels.NeighborhoodHash).initialize()
    with pytest.raises(NotImplementedError):
        HadamardCode(base_graph_kernel=(ShortestPath, {"with_labels": False})).initialize()


def test_graph_kernel_dispatch():
    gk = GraphKernel(kernel="HC")
    gk.initialize()
    assert type(gk.kernel_) is HadamardCode and gk.kernel_.base_graph_kernel is None
    gk = GraphKernel(kernel=["HC", "SP"])
    gk.initialize()
    assert gk.kernel_.base_graph_kernel[0] is ShortestPath
    gk = GraphKernel(kernel={"name": "hadamard_code", "n_iter": 3})
    gk.initialize()
    assert gk.kernel_.n_iter == 3
    gk = GraphKernel(kernel=["HC", "EH"])
    gk.initialize()
    assert gk.kernel_.base_graph_kernel[0] is EdgeHistogram
    assert set(GK_FORMS) == {"gk_str", "gk_list_sp", "gk_dict"}


def test_pickle_fitted():
    hc = HadamardCode(n_iter=3).fit(same_width())
    hc2 = pickle.loads(pickle.dumps(hc))
    assert hc2._labels_enum == hc._labels_enum and hc2._width == hc._width == 4
    assert np.array_equal(hc2.X.block.col_idx, hc.X.block.col_idx) and np.array_equal(hc2.X.ids, hc.X.ids)


def test_cabi_symbols():
    assert {"gk_hc_features", "gk_hc_vectors", "gk_selftest_hc_collision"} <= set(_lib.exported_symbols())
