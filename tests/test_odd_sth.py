"""OddSth on the host: the CPU oracle against the real reference's goldens (K and the fitted identities with their C),
label interning and ranks, the reference's errors and quirks, and GraphKernel dispatch.  No GPU is needed."""
import json
import os
import sys
import warnings

import numpy as np
import pytest
from sklearn.exceptions import NotFittedError

from grakel_b200 import Graph, GraphKernel, OddSth
from grakel_b200.kernels import odd_label_tables
from grakel_b200.packing import Block

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import odd_oracle  # noqa: E402
from odd_cases import GRAPH_OBJECT_CASES, cases, error_cases, key_hash  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "odd_sth.npz"))
CASES = {}
for _name, _X, _Y, _p in cases():
    if _name in GRAPH_OBJECT_CASES:
        _X = [Graph(x[0], x[1], {}) for x in _X]
        _Y = None if _Y is None else [Graph(y[0], y[1], {}) for y in _Y]
    CASES[_name] = (_X, _Y, _p)


@pytest.mark.parametrize("name", json.loads(str(G["__cases__"])))
def test_oracle_matches_golden(name):
    X, Y, p = CASES[name]
    h = p.get("h")
    for norm in (0, 1):
        if f"{name}/fit/{norm}" not in G.files:  # RAW_ONLY_CASES
            continue
        assert np.array_equal(odd_oracle.kernel(X, None, h, bool(norm)), G[f"{name}/fit/{norm}"], equal_nan=True)
        if Y is not None:
            assert np.array_equal(odd_oracle.kernel(X, Y, h, bool(norm)), G[f"{name}/transform/{norm}"], equal_nan=True)
    if f"{name}/keys" not in G.files:  # KEYLESS_CASES
        return
    C = odd_oracle.first_counts(odd_oracle.features(X, h))
    assert {key_hash(k): c for k, c in C.items()} == dict(zip(G[f"{name}/keys"].tolist(), G[f"{name}/C"].tolist()))


def test_neighbour_order_is_part_of_the_result():
    assert not np.array_equal(G["order_forward/fit/0"], G["order_reversed/fit/0"])


def test_issue_probes():
    A = np.array([[0, 1, 0], [1, 0, 0], [0, 0, 0]])
    X = [[A, {0: 1, 1: 1, 2: 1}], [A, {0: 1, 1: 2, 2: 3}]]
    assert np.array_equal(odd_oracle.kernel(X), [[35, 9], [9, 7]])
    assert np.array_equal(odd_oracle.kernel([[{0: [1], 1: [0]}, {0: 1, 1: 1, 2: 5}]]), [[16]])


def test_label_tables():
    ids, rank, strs = odd_label_tables([1, 1.0, 2, "b", "a", 1], [0, 3, 5, 6])
    assert strs == ["1", "1.0", "2", "b", "a"]
    assert ids.tolist() == [0, 1, 2, 3, 4, 0]
    # ranked per graph when the whole list cannot be sorted; 1 and 1.0 tie
    assert rank.tolist() == [0, 0, 1, 1, 0, 0]
    for bad in ("a(b", "x,y", "z)"):
        with pytest.raises(NotImplementedError):
            odd_label_tables([1, bad], [0, 2])
    with pytest.raises(NotImplementedError):
        odd_label_tables([(1, 2)], [0, 1])  # str((1, 2)) = "(1, 2)"
    with pytest.raises(TypeError):
        odd_label_tables([1, "a"], [0, 2])


@pytest.mark.parametrize("name", [e[0] for e in error_cases()])
def test_errors_match_golden(name):
    want = json.loads(str(G["__errors__"]))[name]
    _, X, params = next(e for e in error_cases() if e[0] == name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(Exception) as info:
            OddSth(**params).fit(X)
    assert type(info.value).__name__ == want


def test_quirks():
    errors = json.loads(str(G["__errors__"]))
    X = CASES["random"][0]
    est = OddSth().fit(X)
    with pytest.raises(ValueError) as info:
        est.transform(None)
    assert type(info.value).__name__ == errors["transform_none"]
    with pytest.raises(AttributeError, match="_phi_X") as info:
        OddSth(normalize=True).fit(X).transform(X[:2])
    assert type(info.value).__name__ == errors["fit_then_normalized_transform"]
    with pytest.raises(NotFittedError):
        OddSth().fit(X).diagonal()
    with pytest.warns(UserWarning, match="no implemented parallelization for OddSth"):
        OddSth(n_jobs=2).fit(X)
    with pytest.warns(UserWarning, match="Ignoring empty element"):
        OddSth().fit([[]] + X)
    blk = Block([0, 2], [0, 1, 2], [1, 0], None, [1, 1])
    blk.mode = "sp"
    with pytest.raises(NotImplementedError):
        OddSth().fit(blk)
    with pytest.raises(NotImplementedError):
        OddSth().fit([[{0: [1], 1: [0]}, {0: "a(", 1: "b"}]])


def test_dispatch():
    for spec in ("ODD", "odd_sth", {"name": "ODD", "h": 2}):
        gk = GraphKernel(kernel=spec)
        gk.initialize()
        assert isinstance(gk.kernel_, OddSth)
    gk = GraphKernel(kernel={"name": "odd_sth", "h": 3})
    gk.initialize()
    assert gk.kernel_.h == 3
