"""Golden fixture of Propagation / PropagationAttr: K, the draws, the label enumeration and every level's bins from
the real reference (oracle/_ref, GraKeL 0.1.11) -> tests/golden/propagation.npz.

Each case stores its graphs as dense adjacency matrices with integer labels or attribute rows (in their dtype) and,
where given, the user transition matrix; the parameters (JSON); K of fit_transform and, for transform cases, K of
transform; `_u`, `_b` and the enumeration order of the fit; and the bins of every calculate_LSH call in call order
(fit levels, then transform levels; a transform with labels unseen at fit makes two calls per level: the ordinary
vertices, then the vertices hashed with the extended u).  Labels are integers, so the label set's iteration order
does not depend on string hashing.  Cases with a callable metric (`min_metric`) pin the Counter route; the edge
dictionary case keeps its raw input in the metadata; the error cases record the reference's exception type and
message (a sparse transition matrix, M="H" over a negative entry).

    python tests/golden/make_golden_propagation.py
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))


def mutag(lo, hi):
    sys.path.insert(0, HERE)
    import gio
    X = gio.dec_dataset(gio.load(os.path.join(HERE, "mutag_graphs.json.gz")))[lo:hi]
    out = []
    for g, L in (x[:2] for x in X):
        A, lab = _adjacency(g, L)
        out.append((A, lab, None))
    return out


def _adjacency(g, L):
    from grakel.graph import Graph
    G = Graph(g, L, {}, "adjacency")
    A = np.asarray(G.get_adjacency_matrix(), dtype=float)
    lab = G.get_labels(purpose="adjacency")
    return A, [lab[i] for i in range(A.shape[0])]


def generated(seed, features, n_graphs=30, n_test=10):
    """The reference's own test setup (test_Kernel.py:669-703): real edge weights, a label unseen at fit in every
    transformed graph (features=('nl', k)) or k-dimensional attributes (('na', k))."""
    from grakel.datasets.testing import generate_dataset
    train, test = generate_dataset(n_graphs=n_graphs, r_vertices=(10, 20), r_connectivity=(0.4, 0.8),
                                   r_weight_edges=(1e-5, 10), n_graphs_test=n_test, random_state=seed,
                                   features=features)
    conv = lambda G: [(np.asarray(_adjacency(g[0], g[1])[0]), _adjacency(g[0], g[1])[1], None) for g in G]
    return conv(train), conv(test)


def synthetic(seed, n_graphs, labels=3, signed=False, directed=False, loops=False, user_T=False, single=False):
    rs = np.random.RandomState(seed)
    out = []
    for g in range(n_graphs):
        n = 1 if single and g % 3 == 0 else int(rs.randint(2, 9))
        A = (rs.rand(n, n) < 0.4).astype(float)
        if not directed:
            A = np.triu(A, 1)
            A = A + A.T
        elif not loops:
            np.fill_diagonal(A, 0)
        if loops:
            A[np.diag_indices(n)] = rs.rand(n) < 0.3
        if signed:
            W = rs.choice([0.5, 1.0, 2.0, -1.0, -0.25, 3.0], size=(n, n))
            A = A * W
        if n >= 4:  # an isolated vertex: a zero row of T
            A[n - 1, :] = 0
            A[:, n - 1] = 0
        T = None
        if user_T:
            T = rs.rand(n, n) * (rs.rand(n, n) < 0.6)
            if n >= 3:
                T[0, :] = 0
        out.append((A, [int(rs.randint(labels)) for _ in range(n)], T))
    return out


def with_attrs(G, seed, d, dtype):
    rs = np.random.RandomState(seed)
    out = []
    for A, _, T in G:
        n = A.shape[0]
        if np.dtype(dtype).kind == "i":
            P = rs.randint(-6, 7, size=(n, d)).astype(dtype)
        else:
            P = (rs.rand(n, d) * 4 - 1).astype(dtype)
        out.append((A, [P[i] for i in range(n)], T))
    return out


def min_metric(x, y):
    """A callable metric for the golden cases: the histogram intersection of two levels' Counters."""
    return sum(min(x[k], y[k]) for k in x if k in y)


def cuneiform(lo, hi):
    """Graphs of the reference's bundled Cuneiform (tests/golden/tu) with their node attributes."""
    import tempfile
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    from make_golden_tu import unpack
    from oracle.gk_oracle import read_data_oracle
    d = tempfile.mkdtemp()
    unpack("Cuneiform", d)
    graphs, _ = read_data_oracle(d, "Cuneiform", prefer_attr_nodes=True)
    out = []
    for g, L in (list(x[:2]) for x in graphs[lo:hi]):
        A, lab = _adjacency(g, L)
        out.append((A, [np.asarray(a, dtype=float) for a in lab], None))
    return out


def edge_dicts():
    """Directed weighted edge dictionaries whose symbols are not 0..n-1, with vertices that only appear as targets
    or as self-loops, and negative weights (raw reference input; the adjacency is the reference's)."""
    raw = [
        [[[0, 3, 1.5], [3, 7, -0.5], [7, 0, 2.0], [9, 9, 1.0]], {0: 1, 3: 2, 7: 1, 9: 0}],
        [[[2, 5, 1.0], [5, 2, 1.0], [5, 8, 3.0]], {2: 0, 5: 0, 8: 2}],
        [[[1, 4, 0.25], [4, 6, 1.0], [6, 1, -1.0], [11, 4, 2.0]], {1: 1, 4: 2, 6: 2, 11: 1}],
        [[[0, 1, 1.0]], {0: 2, 1: 2}],
    ]
    return raw


def raw_input(raw):
    return [[{(int(u), int(v)): w for u, v, w in e}, {int(k): v for k, v in dict(L).items()}] for e, L in raw]


def cases():
    m_fit, m_test = mutag(0, 40), mutag(40, 60)
    gen_fit, gen_test = generated(11, ("nl", 4))
    two_new = [(A, [l if l < 4 else 4 + (i % 2) for i, l in enumerate(lab)], T) for A, lab, T in gen_test]
    ga_fit, ga_test = generated(13, ("na", 5))
    sym = synthetic(1, 12)
    dirw = synthetic(2, 12, signed=True, directed=True, loops=True)
    userT = synthetic(3, 10, user_T=True)
    single = synthetic(4, 9, single=True)
    C = []
    add = lambda name, cls, params, X, Y=None, extra=None: C.append((name, cls, params, X, Y, extra or {}))
    add("mutag_tv", "PR", dict(random_state=0), m_fit, m_test)
    add("mutag_h_norm", "PR", dict(random_state=5, M="H", t_max=3, w=1e-4, normalize=True), m_fit, m_test)
    add("mutag_t1_w1", "PR", dict(random_state=2, t_max=1, w=1.0), m_fit, m_test)
    add("generated_new_label", "PR", dict(random_state=3), gen_fit, gen_test)
    add("generated_two_new_labels", "PR", dict(random_state=4, normalize=True), gen_fit, two_new)
    add("generated_new_label_h", "PR", dict(random_state=6, M="H", t_max=3), gen_fit, gen_test)
    add("user_transition", "PR", dict(random_state=7, t_max=3, w=1.0), userT[:7], userT[7:])
    add("directed_signed", "PR", dict(random_state=8), dirw[:8], dirw[8:])
    add("single_vertices", "PR", dict(random_state=9, t_max=3), single)
    add("w_negative", "PR", dict(random_state=10, w=-0.5, t_max=3), sym[:8], sym[8:])
    add("randomstate_object", "PR", dict(random_state="RandomState(12)", t_max=3), sym[:8], sym[8:])
    add("second_fit", "PR", dict(random_state=14, t_max=3), sym, None, {"second_fit": True})
    add("graphkernel_pr", "GK", dict(kernel="PR", random_state=15, normalize=True), sym[:8], sym[8:])
    add("attr_generated_l1", "PRA", dict(random_state=16), ga_fit, ga_test)
    add("attr_generated_l2_norm", "PRA", dict(random_state=17, M="L2", w=0.5, t_max=3, normalize=True), ga_fit, ga_test)
    add("attr_float32", "PRA", dict(random_state=18, w=0.25), with_attrs(dirw[:8], 1, 3, np.float32),
        with_attrs(dirw[8:], 2, 3, np.float32))
    add("attr_int", "PRA", dict(random_state=19, w=1.5, t_max=4), with_attrs(sym[:8], 3, 2, np.int64),
        with_attrs(sym[8:], 4, 2, np.int64))
    add("attr_user_transition", "PRA", dict(random_state=20, t_max=3, w=2.0), with_attrs(userT[:7], 5, 4, np.float64),
        with_attrs(userT[7:], 6, 4, np.float64))
    add("graphkernel_pr_attr", "GK", dict(kernel={"name": "PR", "with_attributes": True}, random_state=21),
        with_attrs(sym[:8], 7, 3, np.float64), with_attrs(sym[8:], 8, 3, np.float64))
    add("metric_callable", "PR", dict(random_state=22, t_max=3), gen_fit, gen_test, {"metric": "min"})
    add("metric_callable_attr", "PRA", dict(random_state=23, t_max=3, normalize=True), ga_fit, ga_test,
        {"metric": "min"})
    add("metric_callable_norm", "PR", dict(random_state=24, normalize=True), m_fit, m_test, {"metric": "min"})
    add("attr_cuneiform_l1", "PRA", dict(random_state=25, w=0.5), cuneiform(0, 30), cuneiform(30, 40))
    add("attr_cuneiform_l2", "PRA", dict(random_state=26, M="L2", t_max=3, normalize=True), cuneiform(0, 30),
        cuneiform(30, 40))
    ed = edge_dicts()
    add("edge_dicts", "PR", dict(random_state=27, t_max=4), ed[:3], ed[3:], {"raw": True})
    add("error_sparse_transition", "PR", dict(random_state=28, t_max=3), userT[:3], None, {"err": "sparse"})
    neg = [(np.array([[0., -1., 0.], [1., 0., 1.], [0., 1., 0.]]), [1, 2, 1], None)]
    add("error_h_negative", "PR", dict(random_state=29, M="H", t_max=3), neg, None, {"err": "run"})
    return C


def as_input(G, extra=None):
    if extra and extra.get("raw"):
        return raw_input(G)
    if extra and extra.get("err") == "sparse":
        import scipy.sparse as sp
        return [[A, dict(enumerate(lab)), {}, sp.csr_matrix(A)] for A, lab, _ in G]
    return _as_input(G)


def _as_input(G):
    """[A, {index: label or attribute row}] or [A, labels, {}, T] per graph: the reference's element spellings."""
    out = []
    for A, lab, T in G:
        el = [A, dict(enumerate(lab))]
        if T is not None:
            el += [{}, T]
        out.append(el)
    return out


def flat(G):
    sizes = np.array([A.shape[0] for A, _, _ in G], dtype=np.int64)
    A = np.concatenate([A.ravel() for A, _, _ in G]) if G else np.zeros(0)
    hasT = np.array([T is not None for _, _, T in G], dtype=bool)
    T = np.concatenate([T.ravel() for _, _, T in G if T is not None] + [np.zeros(0)])
    lab = [l for _, L, _ in G for l in L]
    L = np.stack(lab) if lab and isinstance(lab[0], np.ndarray) else np.array(lab, dtype=np.int64)
    return sizes, A, hasT, T, L


def unflat(sizes, A, hasT, T, L):
    out, a, t, v = [], 0, 0, 0
    for n, h in zip(sizes.tolist(), hasT.tolist()):
        M = A[a:a + n * n].reshape(n, n)
        a += n * n
        U = None
        if h:
            U = T[t:t + n * n].reshape(n, n)
            t += n * n
        lab = [L[i] for i in range(v, v + n)] if L.ndim == 2 else L[v:v + n].tolist()
        v += n
        out.append((M, lab, U))
    return out


def make_estimator(cls, params, extra):
    from grakel import GraphKernel
    from grakel.kernels import Propagation, PropagationAttr
    p = dict(params)
    if extra.get("metric") == "min":
        p["metric"] = min_metric
    if p.get("random_state") == "RandomState(12)":
        p["random_state"] = np.random.RandomState(12)
    if cls == "GK":
        return GraphKernel(**p)
    return (Propagation if cls == "PR" else PropagationAttr)(**p)


def run_reference(cls, params, X, Y, extra):
    est = make_estimator(cls, params, extra)
    kern = est
    calls = []

    def hook(k):
        orig = type(k).calculate_LSH

        def rec(self_, P, u, b):
            h = orig(self_, P, u, b)
            calls.append(np.array(h, dtype=np.float64))
            return h
        k.calculate_LSH = rec.__get__(k)

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if cls == "GK":
            est.initialize()
            kern = est.kernel_
        hook(kern)
        if extra.get("err"):
            try:
                est.fit_transform(as_input(X, extra))
            except Exception as e:  # noqa: BLE001
                return dict(err=[type(e).__name__, str(e)], calls=[], n_fit_calls=0)
            raise AssertionError("no error")
        K = est.fit_transform(as_input(X, extra))
        if extra.get("second_fit"):
            calls.clear()
            K = est.fit_transform(as_input(X, extra))
        n_fit_calls = len(calls)
        u, b = np.stack(kern._u), np.stack([np.atleast_1d(x) for x in kern._b])
        enum = [int(l) for l in kern._enum_labels] if not kern.attr_ else []
        enum_ids = [int(kern._enum_labels[l]) for l in kern._enum_labels] if not kern.attr_ else []
        Kt = est.transform(as_input(Y, extra)) if Y is not None else None
    return dict(K=np.asarray(K, dtype=float), Kt=None if Kt is None else np.asarray(Kt, dtype=float), u=u, b=b,
                enum=np.array(enum, dtype=np.int64), enum_ids=np.array(enum_ids, dtype=np.int64),
                calls=calls, n_fit_calls=n_fit_calls)


def main():
    os.environ.setdefault("PYTHONHASHSEED", "0")
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import grakel
    out = {}
    for name, cls, params, X, Y, extra in cases():
        r = run_reference(cls, params, X, Y, extra)
        meta = dict(cls=cls, params=params, extra=extra, n_fit_calls=r["n_fit_calls"], n_calls=len(r["calls"]),
                    reference=grakel.__version__, err=r.get("err"))
        if extra.get("raw"):
            meta["raw_X"], meta["raw_Y"] = X, Y
        out[name + "/meta"] = np.array(json.dumps(meta))
        if "err" in r:
            print(name, "raises", r["err"])
        for tag, G in (("X", X), ("Y", Y)):
            if G is None or extra.get("raw"):
                continue
            for key, val in zip(("sizes", "A", "hasT", "T", "L"), flat(G)):
                out[name + "/" + tag + "_" + key] = val
        for key in ("K", "Kt", "u", "b", "enum", "enum_ids"):
            if r.get(key) is not None:
                out[name + "/" + key] = r[key]
        for i, h in enumerate(r["calls"]):
            out[name + "/call%d" % i] = h
        if "K" in r:
            print(name, r["K"].shape, len(r["calls"]), "calls")
    np.savez_compressed(os.path.join(HERE, "propagation.npz"), **out)


if __name__ == "__main__":
    main()
