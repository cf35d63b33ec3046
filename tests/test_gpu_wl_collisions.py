"""The WL relabel's collision check and retry, on every relabel route, against the oracle.

Every route hashes a vertex signature (own label, degree, sorted neighbour labels), compares the full signature with the
one its hash slot stands for, raises DevScalars::collision on a mismatch, and the host repeats the pass with a new seed.
gk_selftest_wl_collision makes the next attempts hash (own label, degree) only from a chosen level on, so vertices with
equal label and degree but different neighbours share a slot and only the verification can separate them: the "twins"
of tests/wl_twins.py differ in exactly one sorted position, at the degrees where the kernels change how they sort, store
and compare a signature.  A natural collision at the shipped seed (tests/wl_hash_ref.py) checks the same path without the
hook."""
import functools
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)

import wl_twins as tw  # noqa: E402
from oracle.gk_oracle import WLOAOracle, WLOracle, gen, wl_partitions  # noqa: E402

pytestmark = pytest.mark.gpu

ROUTES = {
    "default": {},  # wl_fused2, slot payloads, resident tiles
    "payload0": {"GRAKEL_B200_WL_PAYLOAD": "0"},  # wl_fused2, verification against the representative's row
    "multitile": {"GRAKEL_B200_WL_TILES_PER_CTA": "3"},  # wl_fused2, tiles re-staged per level (non-resident)
    "multitile-payload0": {"GRAKEL_B200_WL_TILES_PER_CTA": "3", "GRAKEL_B200_WL_PAYLOAD": "0"},
    "multikernel": {"GRAKEL_B200_WL_FUSED": "0"},  # wl_sig_* + wl_resolve
}
V2_ROUTES = ("default", "payload0", "multitile", "multitile-payload0")


@pytest.fixture(scope="module")
def eng():
    from grakel_b200 import _lib
    return _lib.get_engine()


def _route(monkeypatch, route):
    for k, v in ROUTES[route].items():
        monkeypatch.setenv(k, v)


class _Ref:
    def __init__(self, X, h):
        self.X, self.h, self.N = X, h, len(X)
        self.K, levels = WLOracle(n_iter=h).fit_transform(X, return_levels=True)
        d = np.diagonal(self.K)
        with np.errstate(divide="ignore", invalid="ignore"):
            self.Kn = np.nan_to_num(self.K / np.sqrt(np.outer(d, d)))
        self.parts = wl_partitions(levels)
        self.deg = tw.degrees_of(X)
        self.V = len(self.deg)


@functools.lru_cache(maxsize=None)
def _main():
    """Every twin pair in its three placements, depth-3 twins (a split first at level 3), background from gen."""
    return _Ref(tw.block(depth3=(2, 7, 33), background=gen(300, 18, 3)), 4)


@functools.lru_cache(maxsize=None)
def _isolated(d, pos):
    """One (degree, position) twin pair in its three placements among filler: the only group that splits."""
    return _Ref(tw.block(degrees=(d,), positions=(pos,), background=tw.filler(200)), 1)


@functools.lru_cache(maxsize=None)
def _mix(width):
    return _Ref(tw.degree_mix(width), 3)


def _pack(eng, X, mode="wl"):
    from grakel_b200.packing import label_ids, pack
    b = pack(X, mode, len_ok=lambda m: m >= 2)
    ids, _ = label_ids(b.labels, None)
    eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, ids)
    return b, ids


def _check_labels(eng, ref, st, what):
    for lv in range(1, ref.h + 1):
        dev = eng.wl_labels(lv, ref.V).astype(np.int64)
        assert np.array_equal(dev, ref.parts[lv]), f"{what}: level {lv} labels differ from the oracle"
    assert list(st.level_dims[1:ref.h + 1]) == [int(ref.parts[lv].max()) + 1 for lv in range(1, ref.h + 1)], what


def _check_all(eng, ref, st, what, rect=True):
    K, xd, _ = eng.gram(ref.N)
    assert np.array_equal(K, ref.K), f"{what}: K differs from the oracle"
    assert np.array_equal(xd, np.diagonal(ref.K)), what
    Kn, _, _ = eng.gram(ref.N, normalize=True)
    np.testing.assert_allclose(Kn, ref.Kn, rtol=1e-5, atol=0, err_msg=what)
    if rect:
        nf = ref.N - 7
        Kt, _, _ = eng.gram(ref.N, n_fit=nf)
        assert np.array_equal(Kt, ref.K[nf:, :nf]), f"{what}: rectangular K differs"
    _check_labels(eng, ref, st, what)


# ------------------------------------------------------------------------------------------------ forced collisions
@pytest.mark.parametrize("from_level", [1, 3])
@pytest.mark.parametrize("attempts", [1, 3, 8])
@pytest.mark.parametrize("route", list(ROUTES))
def test_forced_collisions_are_retried_to_the_oracle(eng, monkeypatch, route, attempts, from_level):
    """Every degenerate attempt must be caught (hash_retries == attempts) and the first normal attempt must leave no
    trace of the failed ones: K (square, normalised, rectangular), every level's labels and class counts."""
    _route(monkeypatch, route)
    ref = _main()
    assert tw.first_split_level(ref.parts, ref.deg, from_level) == from_level  # the hook has something to catch
    _pack(eng, ref.X)
    eng.selftest_wl_collision(attempts, from_level)
    st = eng.wl_features(ref.h)
    assert int(st.hash_retries) == attempts, f"{route}: {int(st.hash_retries)} retries for {attempts} degenerate attempts"
    _check_all(eng, ref, st, f"{route} attempts={attempts} from={from_level}")
    assert int(eng.wl_features(ref.h).hash_retries) == 0  # the hook is consumed


@pytest.mark.parametrize("pos", tw.POSITIONS)
@pytest.mark.parametrize("d", tw.DEGREES)
@pytest.mark.parametrize("route", list(ROUTES))
def test_each_twin_position_alone_is_caught(eng, monkeypatch, route, d, pos):
    """One twin pair of degree d differing at one sorted position is the ONLY group whose classes differ from its
    (label, degree) group: the verifier must see that one position (payload labels vs row offset at 6/7, the register
    compare at 8/9, the sig_nbr tail, the last label of wl_resolve's loop), or hash_retries stays 0."""
    _route(monkeypatch, route)
    ref = _isolated(d, pos)
    assert tw.first_split_level(ref.parts, ref.deg, 1) == 1
    _pack(eng, ref.X)
    eng.selftest_wl_collision(1, 1)
    st = eng.wl_features(ref.h)
    assert int(st.hash_retries) == 1, f"{route}: twins of degree {d} differing at the {pos} position were not caught"
    K, _, _ = eng.gram(ref.N)
    assert np.array_equal(K, ref.K)
    _check_labels(eng, ref, st, f"{route} d={d} {pos}")


@pytest.mark.parametrize("attempts", [1, 3])
@pytest.mark.parametrize("width", [8, 16, 32])
def test_multikernel_signature_kernels(eng, monkeypatch, width, attempts):
    """The multi-kernel route with each signature kernel (wl_sig_thread8, wl_sig_small<16>, wl_sig_small<32>) and the
    warp-per-vertex kernel for the vertices above the width, all verified by wl_resolve."""
    _route(monkeypatch, "multikernel")
    ref = _mix(width)
    chosen, n_large = tw.group_width(ref.deg)
    assert chosen == width and n_large > 0
    assert tw.first_split_level(ref.parts, ref.deg, 1) == 1
    _pack(eng, ref.X)
    eng.selftest_wl_collision(attempts, 1)
    st = eng.wl_features(ref.h)
    assert int(st.hash_retries) == attempts
    _check_all(eng, ref, st, f"width {width}")


# ------------------------------------------------------------------------------------------------ the retry budget
@pytest.mark.parametrize("from_level", [1, 3])
@pytest.mark.parametrize("route", list(ROUTES))
def test_retry_budget(eng, monkeypatch, route, from_level):
    """Nine degenerate attempts exhaust the retries: the error names the levels, the handle holds no features (gram
    refuses rather than returning the previous block's K, and the label read-back refuses rather than returning the
    failed attempt's labels), and the next call without the hook is the oracle's."""
    from grakel_b200._lib import GrakelB200Error
    _route(monkeypatch, route)
    ref = _main()
    _pack(eng, ref.X)
    eng.wl_features(ref.h)
    eng.gram(ref.N)  # a valid K of this block exists before the failing call
    eng.selftest_wl_collision(9, from_level)
    with pytest.raises(GrakelB200Error, match="repeated hash collisions") as e:
        eng.wl_features(ref.h)
    mask = int(re.search(r"level mask 0x([0-9a-f]+)", str(e.value)).group(1), 16)
    if route in V2_ROUTES:  # bit = level
        lowest = (mask & -mask).bit_length() - 1
        assert lowest == tw.first_split_level(ref.parts, ref.deg, from_level), hex(mask)
    else:
        assert mask == 1
    with pytest.raises(GrakelB200Error):
        eng.gram(ref.N)
    with pytest.raises(GrakelB200Error, match="no such level"):
        eng.wl_labels(1, ref.V)
    st = eng.wl_features(ref.h)
    assert int(st.hash_retries) == 0
    _check_all(eng, ref, st, f"{route} after the budget", rect=False)


# ------------------------------------------------------------------------------------------------ the asynchronous pass
@pytest.mark.parametrize("delivery", ["host_f64", "library_f32", "device_ptr", "dense_all"])
@pytest.mark.parametrize("attempts", [1, 2])
def test_async_pass_falls_back_on_a_collision(eng, delivery, attempts):
    """gk_wl_gram's asynchronous pass turns the collision flag into GramDyn::bad & 16 and repeats through the
    synchronous route, after its GEMM already wrote K from wrong features into the output: the result, the diagonal and
    the statistics must be the synchronous route's.  The next call without the hook takes the asynchronous pass again."""
    import torch
    ref = _main()
    h, N = ref.h, ref.N
    assert N % 4 == 0  # rows of a device result 16-byte aligned: the asynchronous pass accepts the caller's buffer
    _pack(eng, ref.X)
    dev = torch.full((N, N), -1.0, dtype=torch.float32, device="cuda:%d" % eng.device)
    torch.cuda.synchronize()

    def run():
        if delivery == "host_f64":
            K, xd, st = eng.wl_gram(h, want_diag=True)
        elif delivery == "dense_all":
            K, xd, st = eng.wl_gram(h, want_diag=True, dense_all=True)
        elif delivery == "library_f32":
            _, xd, st = eng.wl_gram(h, out=False, dtype=np.float32, want_diag=True)
            K = eng.fetch(np.empty((N, N), dtype=np.float32))
        else:
            dev.fill_(-1.0)
            torch.cuda.synchronize()
            _, xd, st = eng.wl_gram(h, dtype=np.float32, device_ptr=dev.data_ptr(), want_diag=True)
            K = dev.cpu().numpy()
        return np.asarray(K, dtype=np.float64), xd, st

    run()  # leaves the capacities the asynchronous pass sizes itself by
    K, xd, st = run()
    assert int(st.gemm_launches) == 0, "the asynchronous pass did not run"
    assert np.array_equal(K, ref.K)
    eng.selftest_wl_collision(attempts, 1)
    K, xd, st = run()
    assert int(st.gemm_launches) > 0, "a collision in the asynchronous pass must send it to the synchronous route"
    assert int(st.hash_retries) == attempts - 1
    assert np.array_equal(K, ref.K), f"{delivery}: K after the fallback differs from the oracle"
    assert np.array_equal(xd, np.diagonal(ref.K))
    _check_labels(eng, ref, st, delivery)
    K, xd, st = run()
    assert int(st.gemm_launches) == 0 and int(st.hash_retries) == 0
    assert np.array_equal(K, ref.K) and np.array_equal(xd, np.diagonal(ref.K))


# ------------------------------------------------------------------------------------------------ consumers
@pytest.mark.parametrize("route", ["default", "multitile", "payload0"])
def test_wl_oa_after_retries(eng, monkeypatch, route):
    """WL-OA re-adds the frozen vertices' self similarity (diag_frozen), which the failed attempts also wrote."""
    _route(monkeypatch, route)
    X = tw.block(degrees=(1, 2, 7, 9, 33), depth3=(2,), background=gen(60, 12, 4))
    h = 3
    Ko = WLOAOracle(n_iter=h).fit_transform(X)
    _pack(eng, X, mode="wloa")
    eng.selftest_wl_collision(3, 1)
    st = eng.wl_oa_features(h)
    assert int(st.hash_retries) == 3
    K, xd, _ = eng.gram(len(X))
    assert np.array_equal(K, Ko)
    assert np.array_equal(xd, np.diagonal(Ko))


@pytest.mark.parametrize("name", ["er60", "er25_deep"])
def test_level_dictionaries_after_retries(eng, name):
    """The reference's per-level dictionaries rebuilt from a retried relabelling equal the real reference's."""
    import gzip
    import json
    from grakel_b200 import WeisfeilerLehman
    from grakel_b200.kernels import wl_reference_dictionaries
    with gzip.open(os.path.join(HERE, "golden", "inv_labels.json.gz"), "rt") as f:
        case = json.load(f)[name]
    c = case["params"]
    X = gen(c["N"], c["nbar"], c["seed"], nl=c["nl"])
    wl = WeisfeilerLehman(n_iter=c["n_iter"]).fit(X)
    block, ids = wl.X.block, wl.X.ids
    eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids)
    L = c["n_iter"] + 1  # levels 0 .. n_iter
    eng.selftest_wl_collision(2, 1)
    st = eng.wl_features(L - 1)
    assert int(st.hash_retries) == 2
    classes = [ids] + [eng.wl_labels(lv, block.n_vertices) for lv in range(1, L)]
    out, _ = wl_reference_dictionaries(np.asarray(block.row_ptr), np.asarray(block.col_idx), ids, len(wl.X.dictionary),
                                       classes)
    assert sorted(out) == list(range(1, L))
    for i, pairs in case["levels"].items():
        if int(i):
            assert out[int(i)] == {key: v for key, v in pairs}, f"level {i}"


# ------------------------------------------------------------------------------------------------ a natural collision
def test_natural_collision_at_the_shipped_seed(eng):
    """Two star centres whose level-1 keys share the 31-bit tag and the start slot at the first seed (found by the NumPy
    restatement of the hash, tests/wl_hash_ref.py): the table routes them to one slot, the verification must tell them
    apart and the retry must give the oracle's answer -- through gk_wl_features and through gk_wl_gram, whose
    asynchronous pass uses the same first seed and whose synchronous fallback then retries once."""
    import wl_hash_ref
    (oa, na), (ob, nb) = wl_hash_ref.find_colliding_pair()
    labels = [oa] + na + [ob] + nb  # two stars: centre 0 / 9, eight leaves each; raw label ids < 64
    graph_ptr = [0, 9, 18]
    row_ptr, col = [0], []
    for c in (0, 9):
        col += list(range(c + 1, c + 9))
        row_ptr.append(len(col))
        for v in range(c + 1, c + 9):
            col.append(c)
            row_ptr.append(len(col))
    X = []
    for c, own, leaves in ((0, oa, na), (9, ob, nb)):
        g = {}
        for j in range(1, 9):
            g[(0, j)] = g[(j, 0)] = 1
        X.append([g, {0: own, **{j: leaves[j - 1] for j in range(1, 9)}}])
    ref = _Ref(X, 1)
    eng.pack(graph_ptr, row_ptr, col, labels)
    drift = ("no collision: tests/wl_hash_ref.py no longer restates the key, slot or tag of wl_fused2 at the first "
             "seed -- update it with the kernel")
    st = eng.wl_features(1)
    assert int(st.hash_retries) == 1, drift
    K, _, _ = eng.gram(2)
    assert np.array_equal(K, ref.K)
    _check_labels(eng, ref, st, "natural collision")
    K, _, st = eng.wl_gram(1)
    assert int(st.gemm_launches) > 0 and int(st.hash_retries) == 1, drift
    assert np.array_equal(K, ref.K)
