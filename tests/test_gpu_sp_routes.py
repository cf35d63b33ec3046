"""The shortest-path feature routes of sp_features_impl at their dispatch edges (BFS word and thread classes, the
direct table past dcap, the hashed table's fall-through, Floyd-Warshall in shared and global memory, the switch to
real mode, both path-sum orders, table regrowth, KEEP_DIST), through the estimators and the C-ABI, against the float64
reference of sp_routes_ref.py: every integer K bit for bit, normalised K within 1e-14 relative, and stats_.n_columns
equal to the reference's number of distinct features."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import sp_routes_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = R.cases()


def _eq(a, b):
    a = np.asarray(a)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(a, b.astype(np.float64)), (a - b)[np.nonzero(a != b)][:5]


def _close(a, b):
    with np.errstate(all="ignore"):
        np.testing.assert_allclose(np.asarray(a), b, rtol=1e-14, atol=0, equal_nan=True)


def _estimator(c, normalize):
    import grakel_b200 as k
    if c["est"] == "wlsp":
        return k.WeisfeilerLehman(n_iter=c["n_iter"], base_graph_kernel=k.ShortestPath, normalize=normalize)
    if c["est"] == "hcsp":
        return k.HadamardCode(n_iter=c["n_iter"], base_graph_kernel=(k.ShortestPath, {}), normalize=normalize)
    return k.ShortestPath(with_labels=c.get("with_labels", True), algorithm_type=c.get("algorithm_type", "auto"),
                          normalize=normalize)


def _diag_free(c, r):
    # WL over ShortestPath: the fit diagonal follows the reference's own rule (the WL-SP goldens of test_gpu_parity
    # and test_next_rows pin it); every pair entry and the transform matrix are the plain feature-map product
    return c["est"] == "wlsp"


@pytest.mark.parametrize("c", CASES, ids=[c["id"] for c in CASES])
def test_route_case(c, monkeypatch):
    from grakel_b200 import _lib
    for k, v in c.get("env", {}).items():
        monkeypatch.setenv(k, v)
    r = R.reference(c["X"], c["Y"], **R.case_args(c))
    missing = c["expect"] - (R.case_routes(c, r) | R.data_routes(c, r))
    assert not missing, f"the case no longer reaches {missing}"
    off = ~np.eye(len(c["X"]), dtype=bool) if _diag_free(c, r) else np.ones((len(c["X"]),) * 2, dtype=bool)

    # the estimator: fit_transform, transform (unseen labels), normalised
    est = _estimator(c, False)
    K = est.fit_transform(c["X"])
    _eq(np.asarray(K)[off], r["K"][off])
    if c["est"] == "sp":
        assert int(est.stats_.n_columns) == r["fit_info"]["n_columns"]
    if c["Y"] is not None:
        _eq(est.transform(c["Y"]), r["Kt"])
        if c["est"] == "sp":
            assert int(est.stats_.n_columns) == r["info"]["n_columns"]
    if not _diag_free(c, r):
        est = _estimator(c, True)
        Kn = est.fit_transform(c["X"])
        _close(Kn, R.normalized(r["K"], r["xdiag"], r["xdiag"]))
        if c["Y"] is not None:
            _close(est.transform(c["Y"]), R.normalized(r["Kt"], r["xdiag"], r["ydiag"]))
    if c["est"] == "hcsp":
        return

    # the C-ABI on a fresh handle (tables start at their initial sizes): the joint Gram, and the distances
    block, order = r["block"], r["order"]
    ls = r["label_sets"]
    e = _lib.Engine(0)
    try:
        ids = None if ls[0] is None else ls[0].astype(np.int32)
        e.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, block.weights)
        if c["est"] == "wlsp":
            st = e.wl_sp_features(c["n_iter"] - 1)
        else:
            st = e.sp_features(with_labels=ids is not None, dijkstra_order=order == "dijkstra")
        Kf, _, _ = e.gram(block.n_graphs, stats=st)
        n_all = block.n_graphs
        free = ~np.eye(n_all, dtype=bool) if _diag_free(c, r) else np.ones((n_all, n_all), dtype=bool)
        _eq(np.asarray(Kf)[free], r["full"][free])
        assert int(st.n_columns) == r["info"]["n_columns"]
        if c["est"] != "sp" or not c["keep"]:
            return
        sizes = np.diff(block.graph_ptr)
        kind = R.weight_kind(block)
        big = any(n > 512 if kind == "unit" else n * n * 8 > R.SMEM_DIST_MAX for n in sizes)
        if big:
            with pytest.raises(NotImplementedError):
                e.sp_features(with_labels=ids is not None, keep_dist=True, dijkstra_order=order == "dijkstra")
            return
        st = e.sp_features(with_labels=ids is not None, keep_dist=True, dijkstra_order=order == "dijkstra")
        for g, D in enumerate(r["info"]["dists"]):
            got = e.sp_distances(g, D.shape[0])
            assert np.array_equal(got.view(np.int64), np.ascontiguousarray(D, dtype=np.float64).view(np.int64)), g
    finally:
        e.close()


def _csr_graphs(seed, n_graphs, n, extra):
    """Directed graphs with a Hamiltonian cycle (every ordered pair at a finite distance) plus `extra` random out-edges
    per vertex, random real weights."""
    rs = np.random.RandomState(seed)
    rows, cols = [], []
    for g in range(n_graphs):
        u = np.concatenate([np.arange(n), np.repeat(np.arange(n), extra)])
        v = np.concatenate([(np.arange(n) + 1) % n, rs.randint(0, n, n * extra)])
        keep = u != v
        pairs = np.unique(np.stack([u[keep], v[keep]], 1), axis=0)
        rows.append(pairs[:, 0] + g * n)
        cols.append(pairs[:, 1] + g * n)
    r, c = np.concatenate(rows), np.concatenate(cols)
    rp = np.zeros(n_graphs * n + 1, dtype=np.int64)
    np.add.at(rp, r + 1, 1)
    return np.arange(n_graphs + 1) * n, np.cumsum(rp), c, rs.rand(len(c)) + 0.05


def test_more_than_2p24_lengths_is_refused():
    """900 directed 143-vertex graphs with random real weights have about 18.3 million distinct path lengths: more
    than the 24-bit distance field of a real-mode feature key holds.  The distance dictionary grows to 2^24 slots and
    then the call fails with a message that names the limit."""
    from grakel_b200 import _lib
    gp, rp, ci, w = _csr_graphs(41, 900, 143, 3)
    e = _lib.Engine(0)
    try:
        e.pack(gp, rp, ci, None, w)
        with pytest.raises(NotImplementedError, match="2\\^24"):
            e.sp_features(with_labels=False)
        # the handle is still usable afterwards
        gp, rp, ci, w = _csr_graphs(42, 3, 10, 1)
        e.pack(gp, rp, ci, None, w)
        st = e.sp_features(with_labels=False)
        block = type("B", (), dict(graph_ptr=gp.astype(np.int32), row_ptr=rp.astype(np.int32),
                                   col_idx=ci.astype(np.int32), weights=w, n_graphs=3))()
        Phi, info = R.features(block, [None], "fw")
        K, _, _ = e.gram(3, stats=st)
        _eq(K, R.gram(Phi))
        assert int(st.n_columns) == info["n_columns"]
    finally:
        e.close()


def test_label_ids_at_the_key_width():
    """Packed label ids go into bits 44-63 and 24-43 of a feature key: ids up to 2^20 - 2 are accepted and exact,
    2^20 labels are refused."""
    from grakel_b200 import _lib
    X = R.gset(43, [30, 45, 20], L=6)
    block = R.prepare(X, None)["block"]
    top = (1 << 20) - 2
    ids = np.array([0, 1, 12345, 1 << 19, top - 1, top])[R.dense_ids(block.labels)].astype(np.int32)
    Phi, info = R.features(block, [ids.astype(np.int64)], "unit")
    e = _lib.Engine(0)
    try:
        e.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, block.weights)
        st = e.sp_features()
        K, _, _ = e.gram(block.n_graphs, stats=st)
        _eq(K, R.gram(Phi))
        assert int(st.n_columns) == info["n_columns"]
        ids[0] = top + 1
        e.pack(block.graph_ptr, block.row_ptr, block.col_idx, ids, block.weights)
        with pytest.raises(NotImplementedError):
            e.sp_features()
    finally:
        e.close()


def test_spattr_refuses_more_than_32768_lengths():
    """ShortestPathAttr keeps 16-bit block ids per vertex pair: 110 directed 20-vertex graphs with random real weights
    (about 41 800 distinct path lengths, fewer than the 65 536-slot dictionary holds) must be refused, not folded."""
    from grakel_b200 import _lib
    gp, rp, ci, w = _csr_graphs(44, 110, 20, 2)
    e = _lib.Engine(0)
    try:
        e.pack(gp, rp, ci, None, w, np.random.RandomState(1).rand(110 * 20, 2))
        with pytest.raises(NotImplementedError, match="32768"):
            e.spattr_features()
    finally:
        e.close()
