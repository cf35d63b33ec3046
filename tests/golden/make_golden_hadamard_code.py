"""Golden fixtures for HadamardCode (grakel/kernels/hadamard_code.py), produced by the REAL reference (oracle/_ref, or
GRAKEL_REF) when this file is run directly.

Stored per case `c`: K of fit_transform (`c__K`) and of transform (`c__Kt`), the diagonals of a normalised transform
(`c__xd`, `c__yd`), the type of the error the reference raised (`c__err`) and, for the cases marked `vec`, the level
vectors the base kernels received (`c__vec<level>`: one row per packed vertex -- every element's labels dictionary in
key order -- zeros where the level has no vector).  `_labels_enum` is pinned (`c__enum_keys`, `c__enum_ids`) for
integer labels only: the order of string labels depends on the hash seed.  The generate_dataset graphs are stored
(`gen8__*`); every other input is rebuilt by `inputs()`.

    python tests/golden/make_golden_hadamard_code.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")
sys.path.insert(0, HERE)

from make_golden_neighborhood_hash import mutag  # noqa: E402

OUT = os.path.join(HERE, "hadamard_code.npz")


def complete(n, labels):
    return [{(u, v): 1 for u in range(n) for v in range(n) if u != v}, {i: labels[i] for i in range(n)}]


def spellings():
    """Every edge-dictionary spelling: labelled vertices outside the edge dictionary, sinks, isolated vertices written
    {u: {}} and {u: []}, and graphs with every vertex a key."""
    return [
        [{(0, 1): 1, (1, 0): 1}, {0: 1, 1: 2, 5: 1}],
        [{0: {1: 1}}, {0: 1, 1: 2}],
        [{0: [1]}, {0: 1, 1: 2}],
        [{(0, 1): 1}, {0: 1, 1: 2}],
        [{0: {1: 1}, 2: {}}, {0: 1, 1: 2, 2: 3}],
        [{0: [1], 2: []}, {0: 1, 1: 2, 2: 3}],
        [[(0, 1), (1, 2), (2, 0)], {0: 3, 1: 1, 2: 2}],
        [[(0, 1, 2.0), (1, 0, 1.0)], {0: 1, 1: 1}],
        [{0: {1: 1, 2: 1}, 1: {2: 1}, 2: {0: 1}}, {2: 2, 0: 1, 1: 3}],
        [{(3, 4): 1, (4, 5): 1, (5, 3): 1, (3, 3): 1}, {5: 1, 4: 1, 3: 2, 9: 3}],
    ]


def directed(seed=3, n_graphs=12):
    """Directed adjacency matrices with self-loops and isolated vertices, integer labels."""
    rs = np.random.RandomState(seed)
    out = []
    for g in range(n_graphs):
        n = int(rs.randint(2, 11))
        A = (rs.rand(n, n) < 0.35).astype(float)
        if g % 2 == 0:
            A[0, 0] = 1.0
        out.append([A, {i: int(rs.randint(5)) for i in range(n)}])
    return out


def same_width(seed=4, n_graphs=10, n_labels=3):
    """Edge dictionaries with labels 0 .. n_labels-1 (W = 4 for 3 and for 4 labels)."""
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n_graphs):
        n = int(rs.randint(3, 9))
        g = {(u, v): 1 for u in range(n) for v in range(n) if u != v and rs.rand() < 0.4}
        g.update({(u, u + 1): 1 for u in range(n - 1)})
        out.append([g, {i: int(rs.randint(n_labels)) for i in range(n)}])
    return out


def weighted(seed=6, n_graphs=10):
    """Real weights: the same graphs as adjacency matrices (Floyd-Warshall path sums) and as dict-of-dicts (Dijkstra)."""
    rs = np.random.RandomState(seed)
    adj, dic = [], []
    for _ in range(n_graphs):
        n = int(rs.randint(3, 9))
        A = (rs.rand(n, n) < 0.5) * np.round(rs.rand(n, n) * 3 + 0.1, 3)
        np.fill_diagonal(A, 0.0)
        L = {i: int(rs.randint(3)) for i in range(n)}
        adj.append([A, L])
        dic.append([{i: {j: float(A[i, j]) for j in range(n) if A[i, j] > 0} for i in range(n)}, dict(L)])
    return adj, dic


def edge_labelled(seed=8, n_graphs=10):
    """Dict-of-dicts graphs with edge labels (the reference hands a {(u, v): w} element's base kernel no edge labels)."""
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n_graphs):
        n = int(rs.randint(2, 8))
        edges = [(u, v) for u in range(n) for v in range(n) if u != v and (rs.rand() < 0.5 or (u, v) == (0, 1))]
        g = {u: {v: 1 for (a, v) in edges if a == u} for u in range(n)}
        out.append([g, {i: int(rs.randint(3)) for i in range(n)}, {e: int(rs.randint(4)) for e in edges}])
    return out


def generated():
    """generate_dataset of the reference's own test data: the transform labels push nl past a power of two."""
    from grakel.datasets.testing import generate_dataset
    return generate_dataset(n_graphs=20, r_vertices=(5, 10), r_connectivity=(0.4, 0.8), r_weight_edges=(1, 1),
                            n_graphs_test=5, random_state=0, features=("nl", 5))


def pack_generated(prefix, X, Y):
    out = {}
    for side, G in (("X", X), ("Y", Y)):
        out["%s__%s_sizes" % (prefix, side)] = np.array([len(g[1]) for g in G], dtype=np.int64)
        out["%s__%s_adj" % (prefix, side)] = np.concatenate([np.asarray(g[0], dtype=np.float64).ravel() for g in G])
        out["%s__%s_labels" % (prefix, side)] = np.concatenate([np.array([g[1][i] for i in range(len(g[1]))], dtype=np.int64)
                                                                for g in G])
    return out


def unpack_generated(prefix, z):
    out = []
    for side in ("X", "Y"):
        sizes, adj, lab = (z["%s__%s_%s" % (prefix, side, k)] for k in ("sizes", "adj", "labels"))
        G, a, b = [], 0, 0
        for n in sizes.tolist():
            G.append([adj[a:a + n * n].reshape(n, n), {i: int(l) for i, l in enumerate(lab[b:b + n].tolist())}])
            a += n * n
            b += n
        out.append(G)
    return out


def inputs(gen):
    """name -> dict(X, Y, n_iter, base ("VH" | ("SP", params) | "EH"), normalize, n_jobs, vec, enum)."""
    mu = mutag()
    gx, gy = gen
    adj, dic = weighted()
    el = edge_labelled()
    wrap = [complete(65, [0] * 65), complete(65, [i % 2 for i in range(65)])]
    c = {}
    for n in range(1, 6):
        c["mutag_n%d" % n] = dict(X=mu[:60], Y=mu[60:80], n_iter=n, enum=True)
    for norm in (False, True):
        t = "_norm" if norm else ""
        c["gen8_vh" + t] = dict(X=gx, Y=gy, n_iter=3, normalize=norm, enum=True)
        c["gen8_sp" + t] = dict(X=gx, Y=gy, n_iter=3, base=("SP", {}), normalize=norm, enum=True)
        c["samew" + t] = dict(X=same_width(), Y=same_width(seed=5, n_graphs=4, n_labels=4), n_iter=3, normalize=norm,
                              enum=True)
    for n in (1, 2, 3):
        c["spell_n%d" % n] = dict(X=spellings(), Y=spellings()[::-1], n_iter=n, vec=True, enum=True)
    c["directed"] = dict(X=directed(), Y=directed(seed=4, n_graphs=5), n_iter=4, vec=True, enum=True)
    c["directed_jobs"] = dict(X=directed(), Y=directed(seed=4, n_graphs=5), n_iter=4, n_jobs=-1)
    c["sp_fw"] = dict(X=adj, Y=adj[:4], n_iter=3, base=("SP", {}))
    c["sp_dj"] = dict(X=dic, Y=dic[:4], n_iter=3, base=("SP", {}))
    c["sp_dj_norm"] = dict(X=dic, Y=dic[:4], n_iter=2, base=("SP", {}), normalize=True)
    c["eh"] = dict(X=el, Y=edge_labelled(seed=9, n_graphs=4), n_iter=3, base="EH")
    c["eh_norm"] = dict(X=el, Y=edge_labelled(seed=9, n_graphs=4), n_iter=2, base="EH", normalize=True)
    c["wrap"] = dict(X=wrap, Y=None, n_iter=13, vec=True, enum=True)
    c["str"] = dict(X=[[g, {k: "ab"[v % 2] for k, v in L.items()}] for g, L in directed()], Y=None, n_iter=3)
    return c


GK_FORMS = {"gk_str": "HC", "gk_list_sp": ["HC", "SP"], "gk_dict": {"name": "HC", "n_iter": 3}}

ERRORS = {
    "err_n0": dict(n_iter=0),
    "err_nfloat": dict(n_iter=1.5),
    "err_base_str": dict(base_graph_kernel="VH"),
    "err_base_params": dict(base_graph_kernel=("VH", {})),
    "err_base_dict": dict(base_graph_kernel=("VH_class", 5)),
    "err_empty": dict(X=[[]]),
    "err_element": dict(X=[5]),
    "err_iterable": dict(X=5),
}


def _ref():
    for p in (os.environ.get("GRAKEL_REF"), os.path.join(ROOT, "oracle", "_ref")):
        if p and os.path.isdir(os.path.join(p, "grakel")):
            sys.path.insert(0, p)
            break
    import grakel
    return grakel


def vector_rows(X, levels):
    """Level dictionaries -> [V, W] rows in packed order (every labels dictionary in key order), zeros where absent."""
    W = len(next(iter(levels[0].values())))
    rows = []
    for x, d in zip(X, levels):
        for k in x[1]:
            rows.append(np.asarray(d[k], dtype=np.int64) if k in d else np.zeros(W, dtype=np.int64))
    return np.array(rows, dtype=np.int64).reshape(-1, W)


def main():
    grakel = _ref()
    from grakel.kernels import EdgeHistogram, HadamardCode, ShortestPath, VertexHistogram

    class Recorder(VertexHistogram):
        seen = []

        def fit_transform(self, X, y=None):
            X = list(X)
            Recorder.seen.append([dict(x[1]) for x in X])
            return super().fit_transform(X)

    warnings.simplefilter("ignore")
    gen = generated()
    out = pack_generated("gen8", list(gen[0]), list(gen[1]))
    gx, gy = unpack_generated("gen8", out)
    for name, spec in inputs((gx, gy)).items():
        base = spec.get("base", "VH")
        if base == "VH":
            bk = Recorder if spec.get("vec") else None
        elif base == "EH":
            bk = EdgeHistogram
        else:
            bk = (ShortestPath, dict(base[1]))
        Recorder.seen = []
        hc = HadamardCode(n_iter=spec["n_iter"], base_graph_kernel=bk, normalize=spec.get("normalize", False),
                          n_jobs=spec.get("n_jobs"))
        try:
            out[name + "__K"] = hc.fit_transform(spec["X"])
        except Exception as e:
            out[name + "__err"] = np.array(type(e).__name__)
            print(name, "error", type(e).__name__, e)
            continue
        if spec.get("vec"):
            for lv, levels in enumerate(Recorder.seen):
                out["%s__vec%d" % (name, lv)] = vector_rows(spec["X"], levels)
        if spec.get("enum"):
            keys = list(hc._labels_enum)
            out[name + "__enum_keys"] = np.array(keys, dtype=np.int64)
            out[name + "__enum_ids"] = np.array([hc._labels_enum[k] for k in keys], dtype=np.int64)
        if spec.get("Y") is not None:
            out[name + "__Kt"] = hc.transform(spec["Y"])
            if spec.get("normalize"):
                xd, yd = hc.diagonal()
                out[name + "__xd"] = np.asarray(xd, dtype=np.float64).ravel()
                out[name + "__yd"] = np.asarray(yd, dtype=np.float64).ravel()
        print(name, out[name + "__K"].shape, float(out[name + "__K"].sum()),
              None if spec.get("Y") is None else float(out[name + "__Kt"].sum()))
    X = same_width()
    for name, form in GK_FORMS.items():
        out[name + "__K"] = grakel.GraphKernel(kernel=form).fit_transform(X)
        print(name, float(out[name + "__K"].sum()))
    for name, kw in ERRORS.items():
        kw = dict(kw)
        X = kw.pop("X", same_width())
        if kw.get("base_graph_kernel") == ("VH_class", 5):
            kw["base_graph_kernel"] = (VertexHistogram, 5)
        try:
            HadamardCode(**kw).fit_transform(X)
            out[name + "__err"] = np.array("")
        except Exception as e:
            out[name + "__err"] = np.array(type(e).__name__)
        print(name, out[name + "__err"])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
