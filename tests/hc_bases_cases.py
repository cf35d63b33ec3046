"""Inputs of the HadamardCode-over-SubgraphMatching / PyramidMatch / NSPD goldens (tests/golden/make_golden_hc_bases.py),
generated from seeds.  The fitted graphs carry 7 labels (a Hadamard width of 8); `same` transforms add label 7 only, so
the width stays 8, and `wide` transforms add 7 and 8, which widens the matrix to 16."""
import numpy as np

from sm_cases import ke_half, ke_neg
from wl_bases_cases import graphs
from wl_sm_cases import adjacency, directed, edge_dicts

N_ITERS = (1, 2, 5)


def fit_set():
    return graphs(6, 6, 17)


def transform_wide():
    return graphs(3, 6, 18, new_labels=True)


def transform_same():
    """Label 8 folded onto 7: a label the fitted graphs lack, at the fitted width."""
    out = []
    for g, L, E in graphs(3, 6, 18, new_labels=True):
        L = {v: min(l, 7) for v, l in L.items()}
        out.append([g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}])
    return out


def ke_int(a, b):
    return 3 if a == b else 1


# name -> (base name, X, {transform name: Y}, base parameters, n_iter values); GRAPH_OBJECT_CASES wrap every element
# in a Graph
def cases():
    X = fit_set()
    Ys = {"same": transform_same(), "wide": transform_wide()}
    out = {"sm_k5": ("SM", X, Ys, {}, N_ITERS)}
    for k in (0, 1, 2, 3, 4):
        out["sm_k%d" % k] = ("SM", X, Ys, {"k": k}, (2,))
    out["sm_decreasing"] = ("SM", X, Ys, {"k": 4, "lw": "decreasing"}, (1, 5))
    out["sm_ke_none"] = ("SM", X, Ys, {"k": 4, "ke": None}, (2,))
    out["sm_kv_none"] = ("SM", X, Ys, {"k": 3, "kv": None}, (1, 2))
    out["sm_ke_int"] = ("SM", X, Ys, {"k": 4, "ke": ke_int}, (2,))
    out["sm_ke_neg"] = ("SM", X, Ys, {"k": 4, "ke": ke_neg}, (2,))
    out["sm_ke_half"] = ("SM", X, Ys, {"k": 4, "ke": ke_half}, (2, 5))
    D = directed(6, 21)
    out["sm_directed"] = ("SM", D[:4], {"same": D[4:]}, {"k": 4}, (1, 2, 5))
    out["sm_adjacency"] = ("SM", adjacency(X), {k: adjacency(Y) for k, Y in Ys.items()}, {"k": 4}, (2,))
    out["sm_edge_dicts"] = ("SM", edge_dicts(X), {k: edge_dicts(Y) for k, Y in Ys.items()}, {"k": 4}, (2,))
    out["sm_graph_objects"] = ("SM", X, Ys, {"k": 3}, (2,))
    out["nspd_default"] = ("NSPD", X, Ys, {}, N_ITERS)
    out["nspd_r1d2"] = ("NSPD", X, Ys, {"r": 1, "d": 2}, (2,))
    out["nspd_adjacency"] = ("NSPD", adjacency(X), {k: adjacency(Y) for k, Y in Ys.items()}, {"r": 1, "d": 2}, (2,))
    # d = 8 exceeds every graph's size: every embedding comes from the dense eig, whose result does not depend on how
    # many ARPACK calls ran before it in the process
    out["pm_labels"] = ("PM", X, Ys, {"d": 8}, N_ITERS)
    out["pm_nolabels"] = ("PM", X, Ys, {"with_labels": False, "d": 8}, (1, 2))
    out["pm_adjacency"] = ("PM", adjacency(X), {k: adjacency(Y) for k, Y in Ys.items()}, {"L": 3, "d": 8}, (2,))
    return out


GRAPH_OBJECT_CASES = {"sm_graph_objects"}


def error_cases():
    """name -> (base name, X, base parameters): inputs the reference refuses; the goldens keep type and message."""
    X = fit_set()
    g, L, E = X[0]
    e0 = next(iter(E))
    return {
        "sm_no_edge_labels": ("SM", [x[:2] for x in X], {}),
        "sm_no_edge_labels_ke_none": ("SM", [x[:2] for x in X], {"ke": None}),
        "sm_missing_edge_label": ("SM", [[g, L, {e: l for e, l in E.items() if e != e0}]] + X[1:], {}),
        "nspd_no_edge_labels": ("NSPD", [x[:2] for x in X], {}),
    }
