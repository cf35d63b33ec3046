"""The u8 head panel of the integer Gram (u8 x u8 -> s32 wgmma) against the bf16 panel it replaces
(GRAKEL_B200_U8=0): both are exact, so every K must be bit-identical between the two, on every route that reaches
the tensor-core GEMM.  Also checks which panel type ran (gk_stats.gemm_elem_bytes: 1 = u8, 2 = bf16)."""
import os
import sys

import numpy as np
import pytest

from oracle.gk_oracle import WLOracle, gen

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _k():
    import grakel_b200
    return grakel_b200


def _both(monkeypatch, fn):
    """fn() with the u8 panel (default) and with GRAKEL_B200_U8=0: (u8 result, bf16 result)."""
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("GRAKEL_B200_U8", mode)
        out[mode] = fn()
    monkeypatch.delenv("GRAKEL_B200_U8")
    return out["1"], out["0"]


def _workload(n):
    from bench import pack_workload
    return pack_workload(n)


# ------------------------------------------------------------------ dense self-test
@pytest.mark.parametrize("n,d,hi", [(300, 200, 255), (777, 1000, 255), (129, 65, 3), (513, 129, 200)])
def test_selftest_u8_gram_matches_integer_matmul(n, d, hi, monkeypatch):
    """Counts up to 255, d not a multiple of 128 and n not a multiple of 256: the u8 tensor-core Gram equals the int64
    C C^T and the bf16 one."""
    from grakel_b200 import _lib
    rs = np.random.RandomState(n * 7 + d)
    C = (rs.rand(n, d) < 0.3) * rs.randint(1, hi + 1, size=(n, d))
    exact = (C.astype(np.int64) @ C.astype(np.int64).T).astype(np.float64)
    e = _lib.Engine(0)
    try:
        (tc8, simt8), (tc16, _) = _both(monkeypatch, lambda: e.selftest_gram(C))
    finally:
        e.close()
    assert np.array_equal(simt8, exact)
    assert np.array_equal(tc8, exact)
    assert np.array_equal(tc16, exact)


# ------------------------------------------------------------------ config 2 through wl_gram
def test_config2_u8_equals_bf16_on_both_routes(monkeypatch):
    """N = 10 000, h = 5: the first pass of a handle is synchronous, the ones after it asynchronous; every pass gives
    the same K in both modes, with the golden sum."""
    from grakel_b200 import _lib
    gp, rp, ci, lab = _workload(10000)
    n = len(gp) - 1

    def run():
        e = _lib.Engine(0)
        try:
            e.pack(gp, rp, ci, lab)
            Ks, stats = [], []
            for _ in range(3):
                _, _, st = e.wl_gram(5, out=False, dtype=np.float32)
                K = np.empty((n, n), dtype=np.float32)
                e.fetch(K)
                Ks.append(K)
                stats.append((int(st.gram_path), int(st.gemm_elem_bytes), int(st.gemm_launches)))
            return Ks, stats
        finally:
            e.close()

    (K8, s8), (K16, s16) = _both(monkeypatch, run)
    assert s8[0][2] > 0 and all(s[2] == 0 for s in s8[1:]), s8  # synchronous, then asynchronous passes
    assert all(s[:2] == (1, 1) for s in s8), s8
    assert all(s[:2] == (1, 2) for s in s16), s16
    for a, b in zip(K8, K16):
        assert np.array_equal(a, b)
        assert float(a.sum(dtype=np.float64)) == 22925628586.0
    assert np.array_equal(K8[0], K8[2])


# ------------------------------------------------------------------ gram variants
@pytest.fixture(scope="module")
def wl3000():
    return _workload(3000)


_VARIANTS = [
    ("default", {}, {}),
    ("dense_all", {}, {"dense_all": True}),
    ("force_T_1", {"GRAKEL_B200_FORCE_T": "1"}, {}),
    ("force_T_8", {"GRAKEL_B200_FORCE_T": "8"}, {}),
    ("force_T_32", {"GRAKEL_B200_FORCE_T": "32"}, {}),
    ("force_T_4096", {"GRAKEL_B200_FORCE_T": "4096"}, {}),
    ("row_range", {}, {"row_range": (300, 1900)}),
    ("transform", {}, {"n_fit": 1800}),
    ("normalize", {}, {"normalize": True}),
    ("cta2_off", {"GRAKEL_B200_CTA2": "0"}, {}),
    ("widen_off", {"GRAKEL_B200_WIDEN": "0"}, {}),
    ("f32_device", {}, {"out": False, "dtype": np.float32}),
]


@pytest.mark.parametrize("name,env,kw", _VARIANTS, ids=[v[0] for v in _VARIANTS])
def test_gram_variants_u8_equal_bf16(wl3000, name, env, kw, monkeypatch):
    from grakel_b200 import _lib
    gp, rp, ci, lab = wl3000
    n = len(gp) - 1
    for k, v in env.items():
        monkeypatch.setenv(k, v)

    def run():
        e = _lib.Engine(0)
        try:
            e.pack(gp, rp, ci, lab)
            e.wl_features(5)
            st = _lib.GkStats()
            K, xd, yd = e.gram(n, stats=st, **kw)
            if K is None:
                K = np.empty((n, n), dtype=np.float32)
                e.fetch(K)
            return K, xd, yd, int(st.gram_path), int(st.gemm_elem_bytes), int(st.n_dense_columns)
        finally:
            e.close()

    r8, r16 = _both(monkeypatch, run)
    assert np.array_equal(r8[0], r16[0])
    assert np.array_equal(r8[1], r16[1])
    assert r8[3] == r16[3]
    if r8[3] == 1:
        assert (r8[4], r16[4]) == (1, 2)
    else:
        assert r8[5] == 0 and (r8[4], r16[4]) == (0, 0)


@pytest.mark.parametrize("tail_fused", ["1", "0"])
def test_asynchronous_pass_u8_equals_bf16(wl3000, tail_fused, monkeypatch):
    """Asynchronous passes with the tail fused into the GEMM epilogue and with the separate tail kernel."""
    from grakel_b200 import _lib
    gp, rp, ci, lab = wl3000
    monkeypatch.setenv("GRAKEL_B200_TAIL_FUSED", tail_fused)

    def run():
        e = _lib.Engine(0)
        try:
            e.pack(gp, rp, ci, lab)
            out = []
            for _ in range(3):
                K, _, st = e.wl_gram(5)
                out.append((K, int(st.gemm_elem_bytes), int(st.gemm_launches)))
            return out
        finally:
            e.close()

    a, b = _both(monkeypatch, run)
    for (K8, eb8, l8), (K16, eb16, l16) in zip(a, b):
        assert np.array_equal(K8, K16)
        assert (eb8, eb16) == (1, 2)
    assert a[-1][2] == 0 and b[-1][2] == 0


# ------------------------------------------------------------------ other integer Grams
def test_shortest_path_and_wl_oa_u8_equal_bf16(monkeypatch):
    k = _k()
    X = gen(400, 18, 5, nl=3)
    sp8, sp16 = _both(monkeypatch, lambda: k.ShortestPath().fit_transform(X))
    assert np.array_equal(sp8, sp16)
    oa8, oa16 = _both(monkeypatch, lambda: k.WeisfeilerLehmanOptimalAssignment(n_iter=4).fit_transform(X))
    assert np.array_equal(oa8, oa16)
    wl8, wl16 = _both(monkeypatch, lambda: k.WeisfeilerLehman(n_iter=3).fit_transform(X))
    assert np.array_equal(wl8, wl16)
    assert np.array_equal(wl8, WLOracle(n_iter=3).fit_transform(X))


# ------------------------------------------------------------------ which panel ran
def _edgeless(counts):
    lab = np.repeat(np.arange(len(counts)), counts)
    n = len(lab)
    return [np.zeros((n, n)), {i: int(x) for i, x in enumerate(lab)}]


@pytest.mark.parametrize("counts,elem", [((255, 3), 1), ((256, 3), 2)], ids=["count255", "count256"])
def test_panel_type_follows_the_largest_count(counts, elem):
    """A count of 255 runs on the u8 panel, a count of 256 on the bf16 one: through the synchronous route and across
    repeated asynchronous passes (after a 256 the handle's passes take bf16 without a detour)."""
    from grakel_b200 import _lib
    from grakel_b200.packing import label_ids, pack
    X = [_edgeless(counts), _edgeless(counts)]
    Ko = WLOracle(n_iter=2).fit_transform(X)
    e = _lib.Engine(0)
    try:
        b = pack(X, "wl")
        ids, _ = label_ids(b.labels, None, sort_new=False)
        e.pack(b.graph_ptr, b.row_ptr, b.col_idx, ids)
        s = e.wl_features(2)
        K, _, _ = e.gram(2, stats=s)
        assert np.array_equal(K, Ko)
        assert (int(s.gram_path), int(s.gemm_elem_bytes)) == (1, elem)
        for rep in range(3):
            K, _, s = e.wl_gram(2)
            assert np.array_equal(K, Ko), rep
            assert (int(s.gram_path), int(s.gemm_elem_bytes)) == (1, elem), rep
            if rep > 0:
                assert int(s.gemm_launches) == 0, "the asynchronous pass was expected to run"
    finally:
        e.close()


def test_async_pass_with_a_new_count_of_256_falls_back():
    """A handle whose last Gram saw counts <= 255 starts its asynchronous pass on the u8 panel; a pass whose data now
    holds a 256 is caught on the device and repeated through the synchronous route on the bf16 panel."""
    from grakel_b200 import _lib
    from grakel_b200.packing import label_ids, pack
    e = _lib.Engine(0)
    try:
        for counts in ((255, 3), (256, 3)):
            X = [_edgeless(counts), _edgeless(counts)]
            Ko = WLOracle(n_iter=2).fit_transform(X)
            b = pack(X, "wl")
            ids, _ = label_ids(b.labels, None, sort_new=False)
            e.pack(b.graph_ptr, b.row_ptr, b.col_idx, ids)
            elem = 1 if max(counts) <= 255 else 2
            for rep in range(2):
                K, _, s = e.wl_gram(2)
                assert np.array_equal(K, Ko), (counts, rep)
                assert int(s.gemm_elem_bytes) == elem, (counts, rep)
            assert int(s.gemm_launches) == 0, "the second pass on the same data was expected to be asynchronous"
    finally:
        e.close()
