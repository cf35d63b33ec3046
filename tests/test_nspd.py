"""NeighborhoodSubgraphPairwiseDistance on the host: the CPython set emulation the device runs, the estimator's
checks and the dispatcher."""
import pickle
import random

import numpy as np
import pytest
from sklearn.base import clone

from grakel_b200 import GraphKernel, NeighborhoodSubgraphPairwiseDistance
from grakel_b200 import _lib


def _sym_sets():
    rng = random.Random(3)
    for size in [0, 1, 2, 5, 6, 7, 20, 40, 100, 300, 1000, 3000]:
        for kind in ("small", "neg", "big", "str"):
            if kind == "small":
                pool = list(range(80))
            elif kind == "neg":
                pool = list(range(-40, 40))
            elif kind == "big":
                pool = [2 ** 61 + rng.randrange(10 ** 6) for _ in range(80)] + [-(2 ** 62), 2 ** 63 + 5]
            else:
                pool = ["v%d" % rng.randrange(10 ** 6) for _ in range(80)]
            items = set()
            while len(items) < min(size, len(pool) ** 2):
                items.add((rng.choice(pool), rng.choice(pool)))
            yield sorted(items, key=repr)


def _check_order(seq):
    got = _lib.nspd_set_order([hash(a) for a, _ in seq], [hash(b) for _, b in seq])
    assert [seq[k] for k in got] == list({t for t in seq})


@pytest.mark.parametrize("seed", range(4))
def test_set_order_matches_interpreter(seed):
    rng = random.Random(seed)
    for seq in _sym_sets():
        rng.shuffle(seq)
        _check_order(seq)
        # chained: a set built by iterating another set, as the reference filters radius r -> 0
        first = list({t for t in seq})
        sub = [t for t in first if rng.random() < 0.6]
        _check_order(sub)


@pytest.mark.parametrize("size", [19660, 19661, 78642, 78643, 78644, 157286, 320000])
def test_set_order_past_the_doubling_resizes(size):
    """Sizes around the table's growth steps: x4 up to 50 000 items (at insert 19 661 into 131 072 slots), x2 above
    (at inserts 78 643, 157 286 and 314 573), each with a chained set built by iterating the first one."""
    rng = random.Random(size)
    pool = list(range(-700, 700))
    items = set()
    while len(items) < size:
        items.add((rng.choice(pool), rng.choice(pool)))
    seq = list(items)
    rng.shuffle(seq)
    _check_order(seq)
    first = list({t for t in seq})
    _check_order(first)
    _check_order([t for t in first if rng.random() < 0.9])


def test_errors_and_warnings():
    with pytest.raises(ValueError, match="r must be a positive integer"):
        NeighborhoodSubgraphPairwiseDistance(r=-1).fit([])
    with pytest.raises(ValueError, match="d must be a positive integer"):
        NeighborhoodSubgraphPairwiseDistance(d=1.0).fit([])
    with pytest.raises(ValueError, match="parsed input is empty"):
        NeighborhoodSubgraphPairwiseDistance().fit([])
    with pytest.raises(TypeError, match="each element of X"):
        NeighborhoodSubgraphPairwiseDistance().fit([[{0: [1], 1: [0]}, {0: 1, 1: 1}]])
    with pytest.raises(TypeError, match="each element of X"):
        NeighborhoodSubgraphPairwiseDistance().fit([5])
    with pytest.warns(UserWarning, match="no implemented parallelization"):
        with pytest.raises(ValueError, match="parsed input is empty"):
            NeighborhoodSubgraphPairwiseDistance(n_jobs=2).fit([])
    with pytest.warns(UserWarning, match="Ignoring empty element on index: 0"):
        with pytest.raises(ValueError, match="parsed input is empty"):
            NeighborhoodSubgraphPairwiseDistance().fit([[]])
    with pytest.raises(NotImplementedError, match="64 levels"):
        NeighborhoodSubgraphPairwiseDistance(r=7, d=8).fit([])


def test_dispatch_pickle_clone():
    gk = GraphKernel(kernel={"name": "NSPD", "r": 2, "d": 1})
    gk.initialize()
    assert isinstance(gk.kernel_, NeighborhoodSubgraphPairwiseDistance)
    assert (gk.kernel_.r, gk.kernel_.d) == (2, 1)
    gk = GraphKernel(kernel="neighborhood_subgraph_pairwise_distance")
    gk.initialize()
    assert isinstance(gk.kernel_, NeighborhoodSubgraphPairwiseDistance)
    k = NeighborhoodSubgraphPairwiseDistance(r=2, d=3, normalize=True)
    k2 = pickle.loads(pickle.dumps(clone(k)))
    assert k2.get_params() == k.get_params()


# ---- the restatement against the real reference's goldens
import json  # noqa: E402
import os  # noqa: E402
import sys  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import nspd_oracle as O  # noqa: E402
from nspd_cases import cases  # noqa: E402

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nspd.npz"))
CASES = {name: (X, Y, p) for name, X, Y, p in cases()}


@pytest.mark.parametrize("name", json.loads(str(G["__cases__"])))
def test_oracle_matches_goldens(name):
    X, Y, p = CASES[name]
    r, d = p.get("r", 3), p.get("d", 4)
    assert np.array_equal(O.vertex_hashes(X, r, d), G[f"{name}/H"])
    for norm in (0, 1):
        assert np.array_equal(O.fit_transform(X, r, d, bool(norm)), G[f"{name}/fit/{norm}"])
        if Y is not None:
            assert np.array_equal(O.transform(X, Y, r, d, bool(norm)), G[f"{name}/transform/{norm}"])


def test_parse_spellings():
    from grakel_b200.kernels import _nspd_graph
    # an edge list as long as its tuples are wide is an edge list, not a matrix
    assert _nspd_graph([(0, 1), (1, 2)], {0: 1, 1: 2, 2: 1}, {(0, 1): 0, (1, 2): 1})[:2] == (3, [(0, 1), (1, 2)])
    assert _nspd_graph({(5, -2): 1, (-2, 5): 1}, {5: 0, -2: 1}, {(5, -2): 0, (-2, 5): 0})[:2] == (2, [(0, 1), (1, 0)])
    with pytest.raises(ValueError, match="labels for edges"):
        NeighborhoodSubgraphPairwiseDistance().fit([[{0: [1], 1: [0]}, {0: 1, 1: 1}, {}]])
    from grakel_b200 import Graph
    with pytest.raises(ValueError, match="labels for edges"):
        NeighborhoodSubgraphPairwiseDistance().fit([Graph({0: [1], 1: [0]}, {0: 1, 1: 1})])
    with pytest.raises(ValueError, match="labels for vertices"):
        NeighborhoodSubgraphPairwiseDistance().fit([[{0: [1], 1: [0]}, {}, {(0, 1): 1}]])
