"""The reference of test_gpu_sp_routes.py pinned on the CPU: it reproduces SPOracle and the committed shortest-path
goldens (MUTAG, fit_transform.json.gz unit / intw / realw, dijkstra_real.npz), and the cases of the GPU file reach
every route of sp_features_impl's dispatch."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import gio  # noqa: E402
import sp_routes_ref as R  # noqa: E402
from oracle.gk_oracle import SPOracle, gen  # noqa: E402

G = os.path.join(HERE, "golden")


def _norm(K, xd, yd=None):
    return R.normalized(K, xd, xd if yd is None else yd)


def _check(X, Y, with_labels, alg, nrm, K_ref, Kt_ref=None):
    r = R.reference(X, Y, with_labels=with_labels, algorithm_type=alg)
    K = _norm(r["K"], r["xdiag"]) if nrm else r["K"]
    with np.errstate(all="ignore"):
        np.testing.assert_allclose(K, K_ref, rtol=1e-14, atol=0, equal_nan=True) if nrm else \
            np.testing.assert_array_equal(K, K_ref)
        if Kt_ref is not None:
            Kt = _norm(r["Kt"], r["xdiag"], r["ydiag"]) if nrm else r["Kt"]
            np.testing.assert_allclose(Kt, Kt_ref, rtol=1e-14, atol=0, equal_nan=True) if nrm else \
                np.testing.assert_array_equal(Kt, Kt_ref)


@pytest.mark.parametrize("tag", ["unit", "intw", "realw"])
def test_reference_matches_fit_transform_goldens(tag):
    d = gio.load(os.path.join(G, "fit_transform.json.gz"))[tag]
    X, Y = gio.dec_dataset(d["X"]), gio.dec_dataset(d["Y"])
    n = 0
    for key, rec in d["out"].items():
        parts = key.split("_")
        if parts[0] != "sp" or "error" in rec:
            continue
        _check(X, Y, parts[1] == "l", "_".join(parts[2:-1]), parts[-1] == "n", rec["fit_transform"],
               rec.get("transform"))
        n += 1
    assert n >= 6


def test_reference_matches_mutag_and_dijkstra_goldens():
    X = gio.dec_dataset(gio.load(os.path.join(G, "mutag_graphs.json.gz")))
    ref = np.load(os.path.join(G, "mutag_out.npz"))
    np.testing.assert_array_equal(R.reference(X)["K"], ref["sp"])
    tr, te = ref["split_train"].tolist(), ref["split_test"].tolist()
    _check([X[i] for i in tr], [X[i] for i in te], True, "auto", True, ref["sp_norm_train"], ref["sp_norm_test"])

    sys.path.insert(0, G)
    from make_golden_dijkstra import gen_real
    d = np.load(os.path.join(G, "dijkstra_real.npz"))
    X = gen_real(40, 12, 21)
    fit, new = X[:30], X[30:]
    for tag, wl in (("lab", True), ("nolab", False)):
        _check(fit, new, wl, "auto", False, d[f"dj_{tag}_K"], d[f"dj_{tag}_Kt"])
        _check(fit, None, wl, "floyd_warshall", False, d[f"fw_{tag}_K"])
    _check(fit, None, True, "auto", True, d["dj_norm_K"])
    # WL over real-weight ShortestPath: the reference's fit diagonal follows a rule of its own (pinned against the
    # device in test_gpu_parity); every pair entry and the transform matrix are the plain feature-map product
    r = R.reference(fit, new, wl_iter=2)
    off = ~np.eye(len(fit), dtype=bool)
    np.testing.assert_array_equal(r["K"][off], d["wlsp_K"][off])
    np.testing.assert_array_equal(r["Kt"], d["wlsp_Kt"])


@pytest.mark.parametrize("as_adj", [False, True])
@pytest.mark.parametrize("with_labels", [True, False])
def test_reference_matches_sp_oracle(as_adj, with_labels):
    X = gen(12, 14, 3, as_adj=as_adj)
    Y = gen(5, 10, 4, nl=9, as_adj=as_adj)
    o = SPOracle(with_labels=with_labels)
    _check(X, Y, with_labels, "auto", False, o.fit_transform(X), o.transform(Y))
    rs = np.random.RandomState(5)  # real weights, directed: both path-sum orders
    W = [R.graph(rs, int(n), directed=True, weights="real", cycle=True, as_dict=not as_adj) for n in (9, 15, 23)]
    for alg in ("auto", "floyd_warshall", "dijkstra"):
        o = SPOracle(with_labels=with_labels, algorithm_type=alg)
        _check(W[:2], W[2:], with_labels, alg, False, o.fit_transform(W[:2]), o.transform(W[2:]))
    enum = {}
    SPOracle(with_labels=with_labels)._counts(W, enum)
    assert R.reference(W, with_labels=with_labels)["info"]["n_columns"] == len(enum)


def test_route_rule():
    assert R.route(64, "unit", 11) == {"bfs_w1", "bfs_direct"}
    assert R.route(65, "unit", 12) == {"bfs_w2", "bfs_hashed"}
    assert R.route(512, "unit", 3) == {"bfs_w8", "bfs_direct"} and R.route(513, "unit", 3) == {"fw_u16_global"}
    assert R.route(143, "int", 3) == {"fw_f64_shared"} and R.route(144, "int", 3) == {"fw_f64_global"}
    assert R.route(144, "real", 3, "dijkstra") == {"real_switch", "real_dj_global"}
    assert R.call_routes([10, 33, 70], "unit", 5) == {"bfs_w1", "bfs_w2", "bfs_direct", "bfs_t64", "bfs_t128"}
    assert (R.dcap(11), R.dcap(7), R.dcap(3)) == (16, 41, 227)


def test_cases_cover_every_route():
    """Size-dependent routes come from the cases' shapes; the data-dependent ones each case declares are asserted from
    the reference when it runs on the device."""
    covered = {}
    for c in R.cases():
        r = R.prepare(c["X"], c["Y"], **R.case_args(c))
        for x in R.case_routes(c, r) | c["expect"]:
            covered.setdefault(x, []).append(c["id"])
    covered.setdefault("real_switch", []).append("test_more_than_2p24_lengths")
    missing = [x for x in R.ROUTES if x not in covered]
    assert not missing, missing
    for x in R.ROUTES:
        print(f"{x:24s} {', '.join(covered[x][:4])}")
