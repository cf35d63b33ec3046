"""Inputs of the WeisfeilerLehman-over-SubgraphMatching goldens (tests/golden/make_golden_wl_sm.py), generated from
seeds: small graphs, so that the reference's per-level SubgraphMatching at k = 5 stays cheap."""
import numpy as np

from sm_cases import ke_half, ke_neg
from wl_bases_cases import graphs

N_ITERS = (1, 2, 5)


def fit_set():
    return graphs(6, 6, 17)


def transform_set():
    """Carries labels the fitted graphs never have."""
    return graphs(3, 6, 18, new_labels=True)


def directed(n, seed):
    """Directed dict-of-dicts graphs with symbol vertices: a sink (only ever a target), a vertex whose edge dictionary
    entry is empty, and a labelled vertex outside the edges."""
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        k = int(rs.randint(4, 7))
        names = ["v%d" % i for i in range(k)]
        g = {u: {} for u in names[:-1]}
        for i in range(k - 1):
            for j in range(k):
                if i != j and rs.rand() < 0.4:
                    g[names[i]][names[j]] = 1
        g[names[0]][names[-1]] = 1  # names[-1] is a sink
        L = {u: int(rs.randint(3)) for u in names}
        L["iso"] = 1  # labelled, outside the edge dictionary
        E = {(u, v): (L[u] + 2 * L[v]) % 3 for u in g for v in g[u]}
        out.append([g, L, E])
    return out


def adjacency(X):
    """The same graphs as adjacency matrices (vertex i is the i-th key of the labels dictionary)."""
    out = []
    for g, L, E in X:
        n = len(L)
        A = np.zeros((n, n))
        el = {}
        for (u, v), l in E.items():
            A[u, v] = 1.0
            el[(u, v)] = l
        out.append([A, {i: L[i] for i in range(n)}, el])
    return out


def edge_dicts(X):
    """The same graphs as dict-of-dicts edge dictionaries."""
    out = []
    for g, L, E in X:
        d = {u: {} for u in L}
        for (u, v) in g:
            d[u][v] = 1
        out.append([d, dict(L), dict(E)])
    return out


# name -> (X, Y, SubgraphMatching parameters, n_iter values); `graph_objects` cases wrap every element in a Graph
def cases():
    X, Y = fit_set(), transform_set()
    out = {"dirac_k5": (X, Y, {}, N_ITERS)}
    for k in (0, 1, 2, 3, 4):
        out["dirac_k%d" % k] = (X, Y, {"k": k}, (2,))
    out["lw_decreasing"] = (X, Y, {"k": 4, "lw": "decreasing"}, (1, 5))
    out["ke_none"] = (X, Y, {"k": 4, "ke": None}, (2,))
    out["kv_none"] = (X, Y, {"k": 3, "kv": None}, (1, 2))
    out["ke_neg"] = (X, Y, {"k": 4, "ke": ke_neg}, (2,))
    out["ke_half"] = (X, Y, {"k": 4, "ke": ke_half}, (2,))
    D = directed(6, 21)
    out["directed"] = (D[:4], D[4:], {"k": 4}, (1, 2, 5))
    out["adjacency"] = (adjacency(X), adjacency(Y), {"k": 4}, (2,))
    out["edge_dicts"] = (edge_dicts(X), edge_dicts(Y), {"k": 4}, (2,))
    out["graph_objects"] = (X, Y, {"k": 3}, (2,))
    return out


GRAPH_OBJECT_CASES = {"graph_objects"}


def error_cases():
    """name -> (X, SubgraphMatching parameters): inputs the reference refuses; the goldens keep type and message."""
    X = fit_set()
    g, L, E = X[0]
    e0 = next(iter(E))
    return {
        "no_edge_labels": ([x[:2] for x in X], {}),
        "no_edge_labels_ke_none": ([x[:2] for x in X], {"ke": None}),
        "empty_edge_labels": ([[x[0], x[1], {}] for x in X], {}),
        "missing_edge_label": ([[g, L, {e: l for e, l in E.items() if e != e0}]] + X[1:], {}),
        "extra_entry": ([x + [None] for x in X], {}),
    }
