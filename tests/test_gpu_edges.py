"""GPU tests at the edges of the engine's numerical contracts (run with -m gpu on an H100).

A. ShortestPathAttr against a float64 Gram of the oracle's feature map, with attributes of mixed sign, where entries
   of K cancel: every entry within 1e-5 relative (1e-9 with GRAKEL_B200_SPATTR_F64=1).
B. The integer exactness bounds of the tensor-core Gram (counts <= 256, self similarities < 2^24) and the u16 / fp32
   transport switch (largest self similarity < 65536), on either side of each bound, through the synchronous route and
   the asynchronous gk_wl_gram pass.  Off-diagonal entries are checked: the diagonal is rewritten from exact u64 self
   similarities and cannot show a bound error.
C. Kernel variants the engine keeps beside its defaults: the caller's device buffer (GK_OUT_DEVICE) with an unaligned
   and an aligned row pitch, the non-TMA fp32 epilogue, the non-TMA mirror and the symmetric tail bucketing."""
import numpy as np
import pytest

from oracle.gk_oracle import SPAttrOracle, WLOracle, gen, read_data_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from grakel_b200 import _lib
    return _lib.get_engine()


def _k():
    import grakel_b200
    return grakel_b200


# ====================================================================== A. ShortestPathAttr where entries cancel
@pytest.fixture(scope="module")
def cuneiform(tmp_path_factory):
    """The first 40 graphs of the reference's bundled Cuneiform (node attributes of both signs) as a packed block read
    from TU files and as the oracle's list of graphs."""
    from make_golden_tu import unpack
    from grakel_b200.datasets import read_tu
    d = str(tmp_path_factory.mktemp("cuneiform"))
    unpack("Cuneiform", d)
    block = read_tu(d, "Cuneiform", kernel="SP", prefer_attr_nodes=True).data
    graphs, _ = read_data_oracle(d, "Cuneiform", prefer_attr_nodes=True)
    return block, [g[:2] for g in graphs]


def _zero_mean(N, nbar, seed, d):
    X = gen(N, nbar, seed, attr=d, as_adj=True)
    for _g, lab in X:
        for v in lab:
            lab[v] = lab[v] - 0.5
    return X


def _paths(N, seed, d):
    """Path-like graphs of 55-60 vertices (a path plus a few chords): ~50 distinct path lengths, so that at d = 32 the
    per-graph feature map does not fit shared memory at once and spattr_accumulate takes several chunks."""
    rs = np.random.RandomState(seed)
    X = []
    for _ in range(N):
        n = int(rs.randint(55, 61))
        A = np.zeros((n, n))
        i = np.arange(n - 1)
        A[i, i + 1] = A[i + 1, i] = 1
        for _c in range(int(rs.randint(0, 3))):
            a, b = sorted(rs.choice(n, 2, replace=False))
            A[a, b] = A[b, a] = 1
        X.append([A, {v: rs.rand(d) - 0.5 for v in range(n)}])
    return X


def _phi(X):
    """Float64 feature map of the oracle (SPAttrOracle._maps) flattened over the sorted union of path lengths."""
    Fs = SPAttrOracle()._maps(X)
    ds = sorted(set().union(*[f.keys() for f in Fs]))
    dd = next(iter(next(f for f in Fs if f).values())).size if ds else 1
    P = np.zeros((len(X), max(len(ds), 1) * dd))
    for g, f in enumerate(Fs):
        for b, dist in enumerate(ds):
            if dist in f:
                P[g, b * dd:(b + 1) * dd] = f[dist].ravel()
    return P


def _within(K, R, scale, rtol, what):
    """|K - R| <= rtol |R| entrywise.  Where R is exactly zero, K must be zero up to rtol times the entry's cancellation
    scale (sum_k |phi_ik| |phi_jk|): exactly zero when the two feature maps have disjoint supports."""
    K, R = np.asarray(K), np.asarray(R)
    assert K.shape == R.shape, what
    assert np.all(np.isfinite(K)), what
    err = np.abs(K - R)
    bound = np.where(R != 0, rtol * np.abs(R), rtol * scale)
    bad = err > bound
    if bad.any():
        rel = err[R != 0] / np.abs(R[R != 0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} entries outside {rtol:g} relative "
                             f"(max relative error {rel.max():.3g})")


def _sp_attr_cases():
    return [("cuneiform", None), ("zero-mean d=1 N=300", (300, 20, 41, 1)), ("zero-mean d=3 N=129", (129, 20, 4, 3)),
            ("zero-mean d=3 N=1", (1, 20, 5, 3)), ("zero-mean d=16 N=127", (127, 20, 6, 16)),
            ("paths d=32 N=129", (129, None, 7, 32))]


@pytest.fixture(scope="module", params=_sp_attr_cases(), ids=lambda c: c[0])
def sp_attr_case(request, cuneiform):
    name, spec = request.param
    if spec is None:
        block, X = cuneiform
    else:
        N, nbar, seed, d = spec
        X = _paths(N, seed, d) if nbar is None else _zero_mean(N, nbar, seed, d)
        block = X
    P = _phi(X)
    return name, block, X, P


@pytest.mark.parametrize("mode", ["default", "fp64"])
def test_shortest_path_attr_where_entries_cancel(sp_attr_case, mode, monkeypatch, eng):
    """Every entry of fit_transform (square), transform (rectangular), the normalised matrix and a row block within the
    contract of the mode against K = Phi Phi^T in float64; K exactly symmetric, self similarities to 1e-12."""
    name, data, X, P = sp_attr_case
    if mode == "fp64":
        monkeypatch.setenv("GRAKEL_B200_SPATTR_F64", "1")
    else:
        monkeypatch.delenv("GRAKEL_B200_SPATTR_F64", raising=False)
    tol = 1e-9 if mode == "fp64" else 1e-5
    k = _k()
    N = len(X)
    R = P @ P.T
    A = np.abs(P) @ np.abs(P).T  # the cancellation scale of every entry
    dg = np.diagonal(R)

    est = k.ShortestPathAttr()
    K = est.fit_transform(data)
    # mixed signs in the feature map take the fp64 CUDA-core Gram (5), non-negative features the 3xTF32 one (4)
    assert int(est.stats_.gram_path) == (5 if mode == "fp64" or (P < 0).any() else 4)
    _within(K, R, A, tol, f"{name} fit_transform")
    assert np.array_equal(K, K.T)
    np.testing.assert_allclose(np.diagonal(K), dg, rtol=1e-12)

    # a row block of the square matrix, from the features the estimator left on the engine
    rb, re_ = (N // 3, N // 3 + max(1, N // 2)) if N > 1 else (0, 1)
    Kr, _, _ = eng.gram(N, row_range=(rb, re_))
    _within(Kr, R[rb:re_], A[rb:re_], tol, f"{name} row block")

    with np.errstate(divide="ignore", invalid="ignore"):
        Rn = R / np.sqrt(np.outer(dg, dg))
        An = A / np.sqrt(np.outer(dg, dg))
    Kn = k.ShortestPathAttr(normalize=True).fit_transform(data)
    ok = dg > 0
    _within(Kn[np.ix_(ok, ok)], Rn[np.ix_(ok, ok)], An[np.ix_(ok, ok)], tol, f"{name} normalised")

    if N > 1 and isinstance(data, list):
        m = N - N // 3
        e = k.ShortestPathAttr()
        e.fit(X[:m])
        Kt = e.transform(X[m:])
        _within(Kt, R[m:, :m], A[m:, :m], tol, f"{name} transform")


def test_tf32_gram_error_bound_on_mixed_signs(sp_attr_case, monkeypatch):
    """The 3xTF32 tensor-core Gram (forced with GRAKEL_B200_SPATTR_F64=0) keeps its error below 1e-6 of each entry's
    cancellation scale sum_k |phi_ik| |phi_jk|.  For non-negative features that scale is K_ij itself, which is what makes
    the tensor-core path meet 1e-5 relative there (with a 10x margin); features of mixed sign take the fp64 Gram."""
    name, data, X, P = sp_attr_case
    monkeypatch.setenv("GRAKEL_B200_SPATTR_F64", "0")
    est = _k().ShortestPathAttr()
    K = est.fit_transform(data)
    assert int(est.stats_.gram_path) == 4
    A = np.abs(P) @ np.abs(P).T
    R = P @ P.T
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(A > 0, np.abs(K - R) / A, np.abs(K - R))
    print(f"{name}: max |err| / sum|phi||phi| = {ratio.max():.3g}")
    assert ratio.max() < 1e-6, ratio.max()


# ====================================================================== B. exactness and transport bounds
def _edgeless(counts):
    """One graph without edges whose vertices carry the labels 0, 1, ... with the given multiplicities: its WL classes
    keep these counts at every level, so n_iter = h (h + 1 levels) multiplies every inner product by h + 1."""
    lab = np.repeat(np.arange(len(counts)), counts)
    n = len(lab)
    return [np.zeros((n, n)), {i: int(x) for i, x in enumerate(lab)}]


def _load(e, X):
    from grakel_b200.packing import label_ids, pack
    b = pack(X, "wl")
    ids, _ = label_ids(b.labels, None, sort_new=False)
    e.pack(b.graph_ptr, b.row_ptr, b.col_idx, ids)
    return b.n_graphs


def _exact(stats):
    """The exact u64 CUDA-core Gram ran (gram_path 2); else the tensor-core path (1, or 3 when every column is in the
    tail)."""
    return int(stats.gram_path) == 2


_BOUNDS = [  # (label counts of each of two identical graphs, WL iterations, K_01, 2 = the exact Gram, 1 = tensor cores)
    ((256, 256, 256, 256, 64, 8, 1, 1, 1), 62, (1 << 24) + 125, 2),  # odd and above 2^24: fp32 cannot hold it
    ((256, 256, 256, 256, 64, 7, 3, 2, 1), 62, (1 << 24) - 127, 1),
    ((257, 3), 2, 3 * (257 * 257 + 9), 2),  # a count above 256 is not exact in bf16
    ((256, 3), 2, 3 * (256 * 256 + 9), 1),
]


@pytest.mark.parametrize("force_T", [None, "1", "4096"])
@pytest.mark.parametrize("counts,h,k01,path", _BOUNDS, ids=["2^24+125", "2^24-127", "count257", "count256"])
def test_exactness_bounds_on_both_routes(counts, h, k01, path, force_T, monkeypatch):
    """Just above a bound the engine must take the exact u64 CUDA-core Gram (gram_path 2), just below it the tensor-core
    Gram (gram_path 1) -- through the estimator, the synchronous route on a fresh handle, and repeated asynchronous passes
    on that handle, where the bound is checked on the device and an exceeded bound makes the pass fall back by itself.
    FORCE_T = 1 puts every column in the dense panel, 4096 every column in the tail's packed words."""
    from grakel_b200 import _lib
    if force_T is not None:
        monkeypatch.setenv("GRAKEL_B200_FORCE_T", force_T)
    X = [_edgeless(counts), _edgeless(counts)]
    Ko = WLOracle(n_iter=h).fit_transform(X)
    assert Ko[0, 1] == k01 and np.all(Ko == k01)

    wl = _k().WeisfeilerLehman(n_iter=h)
    K = wl.fit_transform(X)
    assert np.array_equal(K, Ko), K
    assert _exact(wl.stats_) == (path == 2)

    e = _lib.Engine(0)
    try:
        n = _load(e, X)
        s = e.wl_features(h)
        K, _, _ = e.gram(n, stats=s)
        assert np.array_equal(K, Ko), K
        assert _exact(s) == (path == 2) and int(s.max_count) == max(counts)
        for rep in range(3):
            K, _, s = e.wl_gram(h)
            assert np.array_equal(K, Ko), (rep, K)
            assert _exact(s) == (path == 2), rep
            if path == 2:
                assert int(s.gemm_launches) > 0, "a pass beyond the bound must fall back to the synchronous route"
            elif rep > 0 and force_T != "4096":  # (without a dense column the pass takes the synchronous route by design)
                assert int(s.gemm_launches) == 0, "the asynchronous pass was expected to run"
    finally:
        e.close()


@pytest.mark.parametrize("no_u16", [False, True])
@pytest.mark.parametrize("counts", [(255, 22, 5, 1), (256,)], ids=["65535", "65536"])
def test_u16_transport_switch(counts, no_u16, monkeypatch):
    """VertexHistogram of two identical graphs with sum c^2 = 65535 (moved as u16) and 65536 (moved as fp32): the
    off-diagonal entries are exact, on the synchronous route and on the asynchronous pass (WL with one level)."""
    from grakel_b200 import _lib
    if no_u16:
        monkeypatch.setenv("GRAKEL_B200_NO_U16", "1")
    X = [_edgeless(counts), _edgeless(counts)]
    want = float(sum(c * c for c in counts))
    K = _k().VertexHistogram().fit_transform(X)
    assert np.all(K == want), K
    e = _lib.Engine(0)
    try:
        _load(e, X)
        for rep in range(3):
            K, _, s = e.wl_gram(0)
            assert np.all(K == want), (rep, K)
            assert int(s.max_diag) == want
    finally:
        e.close()


# ====================================================================== C. kernel variants
def test_payload_free_wl_variant_on_the_asynchronous_pass(monkeypatch):
    """GRAKEL_B200_WL_PAYLOAD=0 (the fused WL kernel verifies candidate classes against the representative's CSR row):
    the asynchronous pass gives the synchronous route's matrix, which is the oracle's."""
    from grakel_b200 import _lib
    monkeypatch.setenv("GRAKEL_B200_WL_PAYLOAD", "0")
    X = gen(700, 14, 37)
    Ko = WLOracle(n_iter=3).fit_transform(X)
    e = _lib.Engine(0)
    try:
        n = _load(e, X)
        s = e.wl_features(3)
        K0, _, _ = e.gram(n, stats=s)
        assert np.array_equal(K0, Ko)
        for rep in range(3):
            K, _, s = e.wl_gram(3)
            assert np.array_equal(K, K0), rep
        assert int(s.gemm_launches) == 0, "the asynchronous pass was expected to run"
    finally:
        e.close()


@pytest.fixture(scope="module")
def wl1000(eng):
    X = gen(1000, 14, 23)
    n = _load(eng, X)
    eng.wl_features(3)
    return n


def _device_buffer(rows, ld, dtype):
    import torch
    t = torch.full((rows + 1, ld), float("nan"), dtype=dtype, device="cuda")  # one guard row beyond the result
    torch.cuda.synchronize()
    return t


def _check_device_result(t, K, what):
    rows, cols = K.shape
    A = t.cpu().numpy().astype(np.float64)
    assert np.array_equal(A[:rows, :cols], K), what
    assert np.isnan(A[:rows, cols:]).all(), f"{what}: row padding written"
    assert np.isnan(A[rows]).all(), f"{what}: guard row written"


@pytest.mark.parametrize("pad", [3, 4])
def test_caller_device_buffer(eng, wl1000, pad):
    """K written into a caller's CUDA tensor with the caller's row pitch (GK_OUT_DEVICE): n_fit + 3 (rows not 16-byte
    aligned: the one-CTA kernel with direct stores) and n_fit + 4 (the TMA-store cluster-pair kernel), fp32 and fp64,
    square, rectangular and row-block shapes -- and through gk_wl_gram.  Nothing outside the result is touched."""
    import torch
    n = wl1000
    K64, _, _ = eng.gram(n)
    nf = n - 136
    Kt64, _, _ = eng.gram(n, n_fit=nf)
    rb, re_ = 300, 557
    for dt, tdt in ((np.float32, torch.float32), (np.float64, torch.float64)):
        t = _device_buffer(n, n + pad, tdt)
        eng.gram(n, dtype=dt, device_ptr=t.data_ptr(), ld=n + pad)
        _check_device_result(t, K64, f"square {dt.__name__}")
        t = _device_buffer(n - nf, nf + pad, tdt)
        eng.gram(n, n_fit=nf, dtype=dt, device_ptr=t.data_ptr(), ld=nf + pad)
        _check_device_result(t, Kt64, f"rectangular {dt.__name__}")
        t = _device_buffer(re_ - rb, n + pad, tdt)
        eng.gram(n, dtype=dt, device_ptr=t.data_ptr(), ld=n + pad, row_range=(rb, re_))
        _check_device_result(t, K64[rb:re_], f"row block {dt.__name__}")
    for rep in range(2):
        t = _device_buffer(n, n + pad, torch.float32)
        eng.wl_gram(3, dtype=np.float32, device_ptr=t.data_ptr(), ld=n + pad)
        _check_device_result(t, K64, f"gk_wl_gram pass {rep}")


@pytest.mark.parametrize("n", [260, 1003, 3000])
def test_epilogue_variants_equal_the_default(eng, n, monkeypatch):
    """GRAKEL_B200_NO_TMA_STORE=1 (fp32 K through direct stores), GRAKEL_B200_MIRROR_TMA=0 (the mirrored block through
    row stores) and GRAKEL_B200_TB_SYM=1 (tail lists with row < column only, asynchronous pass): the default fp64 K bit
    for bit -- square, full tiles and the transform shape."""
    X = gen(n, 14, 29)
    _load(eng, X)
    eng.wl_features(3)
    nf = n - 100
    K0, _, _ = eng.gram(n)
    Kf0, _, _ = eng.gram(n, full_tiles=True)
    Kt0, _, _ = eng.gram(n, n_fit=nf)
    assert np.array_equal(K0, Kf0)
    if n == 260:
        assert np.array_equal(K0, WLOracle(n_iter=3).fit_transform(X))
    for name, val in (("GRAKEL_B200_NO_TMA_STORE", "1"), ("GRAKEL_B200_MIRROR_TMA", "0")):
        monkeypatch.setenv(name, val)
        for dt in (np.float64, np.float32):
            K, _, _ = eng.gram(n, dtype=dt)
            assert np.array_equal(K.astype(np.float64), K0), (name, dt)
            K, _, _ = eng.gram(n, dtype=dt, full_tiles=True)
            assert np.array_equal(K.astype(np.float64), K0), (name, dt, "full tiles")
            K, _, _ = eng.gram(n, n_fit=nf, dtype=dt)
            assert np.array_equal(K.astype(np.float64), Kt0), (name, dt, "transform")
        monkeypatch.delenv(name)
    monkeypatch.setenv("GRAKEL_B200_TB_SYM", "1")
    monkeypatch.setenv("GRAKEL_B200_FORCE_T", "8")  # a tail whatever the cost model would choose
    for rep in range(3):
        K, _, s = eng.wl_gram(3)
        assert np.array_equal(K, K0), ("TB_SYM", rep)
    assert int(s.gemm_launches) == 0, "the asynchronous pass was expected to run"
    assert int(s.n_tail_columns) > 0
