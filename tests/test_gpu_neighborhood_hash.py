"""NeighborhoodHash on the device: level codes (gk_nh_labels) and K against the reference's goldens and the NumPy
restatement, bit for bit; the Gram variants (forced head/tail thresholds, the CUDA-core Gram, row blocks, device
output) against the default; symmetry, determinism, GK_DIST."""
import os
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import nh_oracle  # noqa: E402
from grakel_b200 import GraphKernel, NeighborhoodHash, _lib  # noqa: E402
from grakel_b200.packing import Block  # noqa: E402
from test_neighborhood_hash import CASES, GOLDEN, INPUTS, _check_levels, _fits, _state, mg, restated  # noqa: E402

pytestmark = pytest.mark.gpu


def _config2(n):
    from oracle.gk_oracle import gen
    return gen(n, 40, 0)


class _Draws(np.random.RandomState):
    """A RandomState whose `choice` returns given draws: the reference's codes for bits = 32, whose permutation of
    2^32 values would need 32 GB of host memory in a test."""

    def __init__(self, draws):
        super().__init__(0)
        self.draws = draws

    def choice(self, *args, **kwargs):
        return np.asarray(self.draws)


def _device(nh, Y=None):
    """(block, ids, codes, valid, n_fit) of a fitted estimator, optionally joined with a transform input."""
    F = nh.X
    if Y is None:
        return F.block, F.ids, F.codes, F.valid, F.block.n_graphs
    nh._method_calling = 3
    G = nh.parse_input(Y)
    return (Block.concat(F.block, G.block), np.concatenate([F.ids, G.ids + len(F.codes)]),
            np.concatenate([F.codes, G.codes]), np.concatenate([F.valid, G.valid]), F.block.n_graphs)


def _levels_on_device(nh, Y=None):
    block, ids, codes, valid, _ = _device(nh, Y)
    with _lib.engine() as eng:
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, None, None)
        eng.nh_features(nh.R, nh._nh_code, nh.bits, codes, valid)
        return [eng.nh_labels(r, block.n_vertices) for r in range(nh.R)]


def _same_levels(dev, levels):
    for (c, v), level in zip(dev, levels):
        rc, rv = nh_oracle.as_arrays(level)
        assert np.array_equal(v, rv)
        assert np.array_equal(c[v], rc[rv])


@pytest.mark.parametrize("name,spec", CASES, ids=lambda x: str(x))
def test_golden_cases(name, spec):
    X, Y, _ = INPUTS[name]
    t, R, b, rs = spec
    if b > 16:  # the reference's draws for bits = 32 are taken from the fixture
        key = mg.case_key(name, spec)
        nh = NeighborhoodHash(R=R, nh_type=t, bits=b, random_state=_Draws(GOLDEN[key + "__dict_codes"]))
        runs = [(0, nh)]
        nh.fit(X)
        assert list(nh._labels_hash_dict) == GOLDEN[key + "__dict_keys"].tolist()
    else:
        runs = _fits(name, spec)
    for k, nh in runs:
        key = mg.case_key(name, spec, k)
        if k == 0 and b <= 16:  # the estimator's own fit_transform, on a fresh random state
            nh = NeighborhoodHash(R=R, nh_type=t, bits=b, random_state=_state(rs))
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                K = nh.fit_transform(X)
        else:
            K = _refit_kernel(nh, X)
        levels, gp, n_fit = restated(nh)
        dev = _levels_on_device(nh)
        _same_levels(dev, levels)
        _check_levels([[None if not v else int(c) for c, v in zip(*lv)] for lv in dev], key, "fit")
        assert K.dtype == np.float64
        assert np.array_equal(K, GOLDEN[key + "__K_fit"]), np.abs(K - GOLDEN[key + "__K_fit"]).max()
        assert np.array_equal(K, nh_oracle.kernel(levels, gp, n_fit))
        assert np.array_equal(K, K.T)
        if Y is not None:
            levels, gp, n_fit = restated(nh, Y)
            dev = _levels_on_device(nh, Y)
            _same_levels(dev, levels)
            Kt = nh.transform(Y)
            assert np.array_equal(Kt, GOLDEN[key + "__K_tr"]), np.abs(Kt - GOLDEN[key + "__K_tr"]).max()
            assert np.array_equal(Kt, nh_oracle.kernel(levels, gp, n_fit))
            assert nh.diagonal() == (1.0, 1.0)


def _refit_kernel(nh, X):
    """K of the estimator's current fit (a second fit of one RandomState must not draw again)."""
    F = nh.X
    return nh._nh_run(F.block, F.ids, F.codes, F.valid, F.block.n_graphs)


@pytest.fixture(scope="module")
def config2():
    X = _config2(2000)
    out = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for t in ("simple", "count_sensitive"):
            for b in (8, 16):
                nh = NeighborhoodHash(R=3, nh_type=t, bits=b, random_state=0)
                K = nh.fit_transform(X)
                out[(t, b)] = (nh, K)
    return X, out


@pytest.mark.parametrize("t", ["simple", "count_sensitive"])
@pytest.mark.parametrize("b", [8, 16])
def test_config2_prefix_matches_restatement(config2, t, b):
    X, runs = config2
    nh, K = runs[(t, b)]
    levels, gp, n_fit = restated(nh)
    _same_levels(_levels_on_device(nh), levels)
    assert np.array_equal(K, nh_oracle.kernel(levels, gp, n_fit))
    assert np.array_equal(K, K.T)
    # transform: the first 1500 graphs fitted, the rest transformed (unseen labels are impossible here: same alphabet)
    nh2 = NeighborhoodHash(R=3, nh_type=t, bits=b, random_state=1)
    nh2.fit(X[:1500])
    Kt = nh2.transform(X[1500:])
    levels, gp, n_fit = restated(nh2, X[1500:])
    assert np.array_equal(Kt, nh_oracle.kernel(levels, gp, n_fit))


def _engine_run(nh, Y=None, **gram_kw):
    block, ids, codes, valid, n_fit = _device(nh, Y)
    with _lib.engine() as eng:
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, None, None)
        st = eng.nh_features(nh.R, nh._nh_code, nh.bits, codes, valid)
        K, xd, yd = eng.gram(block.n_graphs, n_fit=n_fit, stats=st, **gram_kw)
    return K, xd, yd, st


@pytest.mark.parametrize("transform", [False, True])
def test_gram_variants_equal_default(config2, monkeypatch, transform):
    X, _ = config2
    nh = NeighborhoodHash(R=3, nh_type="count_sensitive", bits=8, random_state=0).fit(X[:1700])
    Y = X[1700:] if transform else None
    K, xd, yd, st = _engine_run(nh, Y)
    assert st.gram_path == 7 and st.n_levels == 3
    assert np.all(xd == 1.0) and (yd is None or np.all(yd == 1.0))
    for T in ("1", "4096"):
        monkeypatch.setenv("GRAKEL_B200_FORCE_T", T)
        assert np.array_equal(_engine_run(nh, Y)[0], K), T
    monkeypatch.delenv("GRAKEL_B200_FORCE_T")
    assert np.array_equal(_engine_run(nh, Y, simt=True)[0], K)
    rows = K.shape[0]
    a, b = rows // 3, rows // 3 + 157
    assert np.array_equal(_engine_run(nh, Y, row_range=(a, b))[0], K[a:b])
    assert np.array_equal(_engine_run(nh, Y, normalize=True)[0], K)
    import torch
    out = torch.full((rows, K.shape[1] + 3), float("nan"), dtype=torch.float64, device="cuda")
    _engine_run(nh, Y, device_ptr=out.data_ptr(), ld=K.shape[1] + 3)
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.array_equal(o[:, :K.shape[1]], K) and np.all(np.isnan(o[:, K.shape[1]:]))


def test_determinism_and_normalize(config2):
    X, runs = config2
    nh, K = runs[("simple", 8)]
    assert np.array_equal(_refit_kernel(nh, X), K)
    nn = NeighborhoodHash(R=3, nh_type="simple", bits=8, random_state=0, normalize=True)
    assert np.array_equal(nn.fit_transform(X), K)
    assert nn.diagonal() == 1.0


def test_dist_unsupported(config2):
    X, runs = config2
    nh, _ = runs[("simple", 8)]
    with pytest.raises(NotImplementedError, match="GK_DIST"):
        _engine_run(nh, dist=True, row_range=(0, len(X)))


def test_star_larger_than_code_space():
    """A star with 3000 leaves (> 2^8 and > 2^3 codes): the large-degree route of the count-sensitive hash."""
    g = {}
    for v in range(1, 3001):
        g[(0, v)] = 1
        g[(v, 0)] = 1
    rs = np.random.RandomState(2)
    X = [[g, {v: int(rs.randint(5)) for v in range(3001)}], [{(0, 1): 1, (1, 0): 1}, {0: 1, 1: 2}]]
    for t, b in (("count_sensitive", 8), ("count_sensitive", 3), ("simple", 8)):
        nh = NeighborhoodHash(R=3, nh_type=t, bits=b, random_state=0)
        K = nh.fit_transform(X)
        levels, gp, n_fit = restated(nh)
        _same_levels(_levels_on_device(nh), levels)
        assert np.array_equal(K, nh_oracle.kernel(levels, gp, n_fit))


def test_bits_64_codes():
    """Codes of the full 64-bit range (bits = 64 through the C-ABI: the reference cannot draw them)."""
    X = INPUTS["many"][0]
    nh = NeighborhoodHash(R=3, nh_type="count_sensitive", bits=16, random_state=0).fit(X)
    rs = np.random.RandomState(9)
    nh.X.codes = rs.randint(0, 2 ** 63, size=len(nh.X.codes), dtype=np.int64).astype(np.uint64) * np.uint64(2) + \
        np.uint64(1)
    for t in ("simple", "count_sensitive"):
        nh.nh_type, nh._nh_code, nh.bits = t, {"simple": 0, "count_sensitive": 1}[t], 64
        levels, gp, n_fit = restated(nh)
        _same_levels(_levels_on_device(nh), levels)
        F = nh.X
        K = nh._nh_run(F.block, F.ids, F.codes, F.valid, F.block.n_graphs)
        assert np.array_equal(K, nh_oracle.kernel(levels, gp, n_fit))


def test_nystroem_over_nh():
    X = _config2(300)
    gk = GraphKernel(kernel={"name": "NH", "R": 3}, Nystroem=40, random_state=0)
    Z = gk.fit_transform(X)
    assert Z.shape == (300, 40) and np.all(np.isfinite(Z))
    assert gk.kernel_.X.block.n_graphs == 40


def test_read_tu_block_equals_list_input():
    from test_neighborhood_hash import _mutag_block
    block = _mutag_block()
    X = mg.mutag()
    for t in ("simple", "count_sensitive"):
        Kb = NeighborhoodHash(R=3, nh_type=t, random_state=0).fit_transform(block)
        Kl = NeighborhoodHash(R=3, nh_type=t, random_state=0).fit_transform(X)
        assert np.array_equal(Kb, Kl), t


def test_packed_block_refuses_order_dependent_codes():
    """A packed block does not carry the reference's neighbour order: a count-sensitive result that depends on it is
    refused; the list input of the same graphs runs and matches the restatement."""
    from grakel_b200.packing import pack
    X = INPUTS["inter"][0]
    block = pack(X, "wl")
    with pytest.raises(NotImplementedError, match="neighbour order"):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            NeighborhoodHash(R=3, nh_type="count_sensitive", bits=1, random_state=0).fit_transform(block)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        nh = NeighborhoodHash(R=3, nh_type="count_sensitive", bits=1, random_state=0)
        K = nh.fit_transform(X)
    assert nh.stats_.nh_order_dependent == 1
    levels, gp, n_fit = restated(nh)
    assert np.array_equal(K, nh_oracle.kernel(levels, gp, n_fit))


def test_row_chunks_equal_one_pass(config2, monkeypatch):
    """The chunked route of the Gram (count matrices above the budget): several row chunks, no mirrored combine."""
    X, runs = config2
    nh, K = runs[("count_sensitive", 16)]
    monkeypatch.setenv("GRAKEL_B200_NH_C_BUDGET", str(3 * 700 * 2000 * 4))  # about 700 rows per chunk
    assert np.array_equal(_refit_kernel(nh, X), K)
    nh2 = NeighborhoodHash(R=3, nh_type="count_sensitive", bits=16, random_state=1).fit(X[:1500])
    Kt = nh2.transform(X[1500:])
    monkeypatch.setenv("GRAKEL_B200_NH_C_BUDGET", str(3 * 1504 * 60 * 4))  # 60 rows per chunk
    assert np.array_equal(nh2.transform(X[1500:]), Kt)
