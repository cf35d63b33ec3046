"""Golden fixtures for GraphHopper (grakel/kernels/graph_hopper.py), produced by the REAL reference (oracle/_ref, or
GRAKEL_REF) when this file is run directly: connected symmetric graphs and directed graphs in which every vertex has
an out-edge (the reference raises on vertices that reach nothing but themselves), all four kernel types,
fit_transform and a transform whose graphs have a larger diameter than the fitted ones, normalised and raw, a few
per-graph node maps, and the first Cuneiform graphs.  Inputs are regenerated from the seeds by `inputs()`; only the
reference's results are stored.

    python tests/golden/make_golden_graph_hopper.py
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..", "..")
KERNEL_TYPES = ("linear", "gaussian", ("gaussian", 0.3), "bridge")


def connected(n_graphs, nbar, seed, dim=3, extra=1.5):
    """Connected symmetric graphs: a random spanning tree plus ER edges; attributes rounded to 3 digits."""
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n_graphs):
        n = int(rs.randint(max(2, nbar // 2), nbar + nbar // 2 + 1))
        A = np.zeros((n, n))
        for v in range(1, n):
            u = int(rs.randint(v))
            A[u, v] = A[v, u] = 1
        iu = np.triu_indices(n, 1)
        m = rs.rand(len(iu[0])) < extra / max(n - 1, 1)
        A[iu[0][m], iu[1][m]] = 1
        A = np.maximum(A, A.T)
        out.append([A, {i: rs.rand(dim).round(3).tolist() for i in range(n)}])
    return out


def paths(n_graphs, n0, seed, dim=3):
    """Path graphs (large diameter) with a few chords."""
    rs = np.random.RandomState(seed)
    out = []
    for k in range(n_graphs):
        n = n0 + 2 * k
        A = np.zeros((n, n))
        A[np.arange(n - 1), np.arange(1, n)] = 1
        A = A + A.T
        out.append([A, {i: rs.rand(dim).round(3).tolist() for i in range(n)}])
    return out


def directed(n_graphs, nbar, seed, dim=2):
    """Directed graphs in which every vertex has an out-edge (a random successor plus sparse extra arcs)."""
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n_graphs):
        n = int(rs.randint(max(3, nbar // 2), nbar + nbar // 2 + 1))
        A = (rs.rand(n, n) < 1.2 / n).astype(float)
        np.fill_diagonal(A, 0)
        for v in range(n):
            w = int(rs.randint(n - 1))
            A[v, w if w < v else w + 1] = 1
        out.append([A, {i: rs.rand(dim).round(3).tolist() for i in range(n)}])
    return out


def inputs():
    """name -> (X, Y or None) of every golden case."""
    return {
        "sym": (connected(14, 9, 1), connected(6, 9, 2)),
        "sym_long": (connected(8, 7, 3, extra=0.5), paths(4, 14, 4)),
        "dir": (directed(12, 8, 5), directed(5, 8, 6)),
    }


def cuneiform():
    """The first 40 graphs of the reference's bundled Cuneiform (tests/golden/tu), with node attributes."""
    import tempfile
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    from make_golden_tu import unpack
    from oracle.gk_oracle import read_data_oracle
    d = tempfile.mkdtemp()
    unpack("Cuneiform", d)
    graphs, _ = read_data_oracle(d, "Cuneiform", prefer_attr_nodes=True)
    return [list(g[:2]) for g in graphs]


def _ref():
    for p in (os.environ.get("GRAKEL_REF"), os.path.join(ROOT, "oracle", "_ref")):
        if p and os.path.isdir(os.path.join(p, "grakel")):
            sys.path.insert(0, p)
            break
    from grakel.kernels import GraphHopper
    return GraphHopper


def _tag(kt):
    return kt if isinstance(kt, str) else "%s_%g" % kt


def main():
    GraphHopper = _ref()
    warnings.simplefilter("ignore")
    out = {}
    for name, (X, Y) in inputs().items():
        for kt in KERNEL_TYPES:
            for norm in (False, True):
                gh = GraphHopper(kernel_type=kt, normalize=norm)
                key = "%s__%s__%d" % (name, _tag(kt), int(norm))
                out[key + "__fit"] = gh.fit_transform(X)
                out[key + "__tr"] = gh.transform(Y)
        gh = GraphHopper(kernel_type="linear")
        gh.fit(X)
        for g in range(3):
            out["%s__M%d" % (name, g)] = gh.X[g][0]
    graphs = cuneiform()
    ok = []
    for i, g in enumerate(graphs):  # the graphs the reference accepts
        try:
            GraphHopper().fit_transform([g])
            ok.append(i)
        except Exception:
            pass
    out["cuneiform__idx"] = np.asarray(ok)
    for kt in KERNEL_TYPES:
        out["cuneiform__%s" % _tag(kt)] = GraphHopper(kernel_type=kt).fit_transform([graphs[i] for i in ok])
    np.savez_compressed(os.path.join(HERE, "graph_hopper.npz"), **out)
    print("wrote", len(out), "arrays")


if __name__ == "__main__":
    main()
