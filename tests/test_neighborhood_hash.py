"""NeighborhoodHash host side (no GPU): validation, the code dictionary and the vertex sets against the reference's
goldens, the NumPy restatement against the goldens bit for bit, pickling and GraphKernel dispatch."""
import os
import pickle
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

import nh_oracle  # noqa: E402
from grakel_b200 import GraphKernel, NeighborhoodHash  # noqa: E402
from grakel_b200.packing import Block  # noqa: E402
import make_golden_neighborhood_hash as mg  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "neighborhood_hash.npz"))
INPUTS = mg.inputs(mg.unpack_generated(GOLDEN))
CASES = [(name, spec) for name, (_, _, specs) in INPUTS.items() for spec in specs]


def _state(rs):
    return np.random.RandomState(rs[1]) if isinstance(rs, tuple) else rs


def _fits(name, spec):
    """(fit number, estimator after that fit) for every fit of a golden case (no device work)."""
    X = INPUTS[name][0]
    t, R, b, rs = spec
    nh = NeighborhoodHash(R=R, nh_type=t, bits=b, random_state=_state(rs))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for k in range(2 if isinstance(rs, tuple) else 1):
            nh.fit(X)
            yield k, nh


def restated(nh, Y=None):
    """(levels, graph_ptr, n_fit) of the restatement on the estimator's packed fit (+ transform) block."""
    F = nh.X
    block, codes0 = F.block, [int(F.codes[i]) if F.valid[i] else None for i in F.ids]
    n_fit = block.n_graphs
    if Y is not None:
        nh._method_calling = 3
        G = nh.parse_input(Y)
        block = Block.concat(block, G.block)
        codes0 = codes0 + [int(G.codes[i]) if G.valid[i] else None for i in G.ids]
    levels = nh_oracle.hash_levels(codes0, block.row_ptr, block.col_idx, nh.R, nh.nh_type, nh.bits)
    return levels, block.graph_ptr, n_fit


def _check_levels(levels, key, side, n_skip=0):
    codes, valid = GOLDEN[key + "__codes_" + side], GOLDEN[key + "__valid_" + side]
    for r, level in enumerate(levels):
        c, v = nh_oracle.as_arrays(level[n_skip:])
        assert np.array_equal(v, valid[r].astype(bool)), (key, side, r)
        assert np.array_equal(c[v], codes[r][v]), (key, side, r)


@pytest.mark.parametrize("name,spec", [c for c in CASES if c[1][2] <= 16], ids=lambda x: str(x))
def test_code_dictionary_matches_reference(name, spec):
    for k, nh in _fits(name, spec):
        key = mg.case_key(name, spec, k)
        d = nh._labels_hash_dict
        assert list(d.keys()) == GOLDEN[key + "__dict_keys"].tolist()
        assert list(d.values()) == GOLDEN[key + "__dict_codes"].tolist()


@pytest.mark.parametrize("name,spec", [c for c in CASES if c[1][2] <= 16], ids=lambda x: str(x))
def test_restatement_matches_reference(name, spec):
    Y = INPUTS[name][1]
    for k, nh in _fits(name, spec):
        key = mg.case_key(name, spec, k)
        levels, gp, n_fit = restated(nh)
        _check_levels(levels, key, "fit")
        assert np.array_equal(nh_oracle.kernel(levels, gp, n_fit), GOLDEN[key + "__K_fit"])
        if Y is not None:
            levels, gp, n_fit = restated(nh, Y)
            _check_levels(levels, key, "tr", n_skip=int(nh.X.block.n_vertices))
            assert np.array_equal(nh_oracle.kernel(levels, gp, n_fit), GOLDEN[key + "__K_tr"])


def test_many_labels_warn_like_the_reference():
    with pytest.warns(UserWarning, match="Number of labels is smaller thanthe biggest possible.. Collisions will "
                                         "appear on the new labels."):
        NeighborhoodHash(bits=3, random_state=1).fit(INPUTS["many"][0])


def test_vertex_set_is_the_edge_dictionary():
    """Vertices are the edge dictionary's symbols (a target-only symbol included); the label of a vertex outside every
    edge only enters the code dictionary; a key with an empty list fails as in the reference."""
    nh = NeighborhoodHash(random_state=0).fit(INPUTS["vset"][0])
    assert np.diff(nh.X.block.graph_ptr).tolist() == [3, 3, 4, 3]
    assert 42 in nh._labels_hash_dict and 17 in nh._labels_hash_dict
    with pytest.raises(ValueError, match="vertex not inside edge dictionary"):
        NeighborhoodHash().fit([[{0: [1], 1: [0], 3: []}, {0: 1, 1: 2, 3: 1}]])


@pytest.mark.parametrize("kw,exc,msg", [
    ({"R": 0}, TypeError, "R must be an intger bigger than zero"),
    ({"R": 2.0}, TypeError, "R must be an intger bigger than zero"),
    ({"nh_type": "other"}, TypeError, "unrecognised neighborhood hashing type"),
    ({"bits": 0}, TypeError, "illegal number of bits for hashing"),
    ({"bits": "8"}, TypeError, "illegal number of bits for hashing"),
    ({"bits": 65}, NotImplementedError, "bits > 64"),
    ({"R": 65}, NotImplementedError, "R = 64"),
])
def test_parameter_validation(kw, exc, msg):
    with pytest.raises(exc, match=msg):
        NeighborhoodHash(**kw).fit(INPUTS["order"][0])


def test_input_validation():
    nh = NeighborhoodHash()
    with pytest.raises(ValueError, match="`fit` input cannot be None"):
        nh.fit(None)
    with pytest.raises(TypeError, match="input must be an iterable"):
        nh.fit(5)
    with pytest.raises(TypeError, match="Labels must be provided"):
        nh.fit([INPUTS["order"][0][0], [{(0, 1): 1}]])
    with pytest.raises(TypeError, match="each element of X must be either a graph object"):
        nh.fit([[{(0, 1): 1}, {0: 1, 1: 2}, {}, {}]])
    with pytest.raises(ValueError, match="Graph does not have any labels for vertices."):
        nh.fit([[{(0, 1): 1}, {}]])
    with pytest.warns(UserWarning, match="Ignoring empty element on index: 0"):
        nh.fit([[]] + INPUTS["order"][0])
    with pytest.raises(ValueError, match="parsed input is empty"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            nh.fit([[]])


def test_diagonal_after_fit():
    nh = NeighborhoodHash(random_state=0).fit(INPUTS["order"][0])
    assert nh.diagonal() == 1.0


def test_pickle_fitted_estimator():
    nh = NeighborhoodHash(R=2, nh_type="count_sensitive", bits=16, random_state=3).fit(INPUTS["many"][0])
    nh2 = pickle.loads(pickle.dumps(nh))
    assert nh2._labels_hash_dict == nh._labels_hash_dict
    assert np.array_equal(nh2.X.codes, nh.X.codes) and np.array_equal(nh2.X.ids, nh.X.ids)
    assert nh2.get_params() == nh.get_params()


def test_graph_kernel_dispatch():
    for name in ("NH", "neighborhood_hash"):
        gk = GraphKernel(kernel={"name": name, "R": 2, "bits": 16, "nh_type": "count_sensitive"}, normalize=True)
        gk.initialize()
        k = gk.kernel_
        assert type(k) is NeighborhoodHash and (k.R, k.bits, k.nh_type, k.normalize) == (2, 16, "count_sensitive", True)
    with pytest.raises(NotImplementedError):
        GraphKernel(kernel="random_walk").initialize()


def _mutag_block():
    import tempfile
    from make_golden_tu import unpack
    from grakel_b200.datasets import read_tu
    d = tempfile.mkdtemp()
    unpack("MUTAG", d)
    return read_tu(d, "MUTAG", kernel="NH").data


def test_read_tu_block_matches_list_input():
    """read_tu(kernel="NH") keeps every labelled node for the code dictionary and walks the edge nodes."""
    block = _mutag_block()
    X = mg.mutag()
    a = NeighborhoodHash(random_state=0).fit(block)
    b = NeighborhoodHash(random_state=0).fit(X)
    assert list(a._labels_hash_dict.items()) == list(b._labels_hash_dict.items())
    assert np.array_equal(np.diff(a.X.block.graph_ptr), np.diff(b.X.block.graph_ptr))
    assert a.X.order_known is False and b.X.order_known is True


def test_neighbours_keep_edge_dictionary_order():
    """The count-sensitive hash depends on the neighbour order of the edge dictionary: rows are not sorted."""
    X = [[{(0, 3): 1, (0, 1): 1, (0, 2): 1, (2, 0): 1, (1, 3): 1}, {0: 1, 1: 2, 2: 1, 3: 2}],
         [np.array([[0, 1, 1], [1, 0, 0], [1, 1, 0]]), {0: 1, 1: 2, 2: 1}]]
    b = NeighborhoodHash(random_state=0).fit(X).X.block
    assert b.col_idx.tolist() == [3, 1, 2, 3, 0, 5, 6, 4, 4, 5]


def test_radix_runs_of_interleaved_codes():
    """bits = 2, neighbour codes [7, 3, 7]: equal low bits, different values, so three runs of one."""
    r = nh_oracle.rot
    assert nh_oracle.radix_sort_rot([7, 3, 7], 2) == r(7 ^ 1, 1, 2) ^ r(3 ^ 1, 1, 2) ^ r(7 ^ 1, 1, 2) == 1
