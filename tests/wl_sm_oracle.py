"""CPU restatement of WeisfeilerLehman over SubgraphMatching (weisfeiler_lehman.py:160-270, 366-482): every level's
labels of the fitted and transformed graphs from the reference's credentials (own label, sorted out-neighbour labels),
numbered jointly (SubgraphMatching with kv=_dirac reads only label equality), every level's elements parsed by
SubgraphMatching.parse_input, the SubgraphMatching restatement (tests/sm_oracle.py) per level, and the levels summed in
level order as np.sum(axis=0) does.  Normalised as WeisfeilerLehman does: by the sum's diagonal after fit_transform, by
the level-ordered sums of the base diagonals after a transform."""
import numpy as np

import sm_oracle
from grakel_b200 import SubgraphMatching
from grakel_b200.packing import adjacency_and_order


def level_elements(X, Y, n_iter):
    """Every level's elements [edges, {vertex: label}, edge labels] of X and of Y (None without Y)."""
    XY = [list(x) for x in list(X) + list(Y or [])]
    nbs = []
    for x in XY:
        A, order = adjacency_and_order(x[0])
        order = list(order)
        nbs.append({order[i]: [order[j] for j in np.flatnonzero(A[i] > 0)] for i in range(len(order))})
    labels = [dict(x[1]) for x in XY]
    out = []
    for h in range(n_iter + 1):
        if h:
            creds = [{v: (L[v], tuple(sorted(L[u] for u in nb.get(v, [])))) for v in L} for L, nb in zip(labels, nbs)]
            ids = {}
            labels = [{v: ids.setdefault(c, len(ids)) for v, c in C.items()} for C in creds]
        els = [[x[0], L] + x[2:] for x, L in zip(XY, labels)]
        out.append((els[:len(X)], els[len(X):] if Y else None))
    return out


def _levels(params, n_iter, X, Y):
    sm = SubgraphMatching(**params)
    sm.initialize()
    out = []
    for lx, ly in level_elements(X, Y, n_iter):
        out.append((sm.parse_input(lx), None if ly is None else sm.parse_input(ly)))
    return sm, out


def kernel(params, n_iter, X, Y=None, normalize=False):
    """K of fit_transform(X), or of transform(Y) after fit(X)."""
    sm, levels = _levels(params, n_iter, X, Y)
    Ks, dx, dy = [], [], []
    for gx, gy in levels:
        Ks.append(sm_oracle.gram(gx, gy, sm.kv, sm.ke, sm.k, sm.lambdas_))
        if Y is not None:
            f = lambda a: sm_oracle.sm_value(a, a, sm.kv, sm.ke, sm.k, sm.lambdas_)
            dx.append(np.array([f(a) for a in gx]))
            dy.append(np.array([f(a) for a in gy]))
    K = np.sum(Ks, axis=0)
    if not normalize:
        return K
    if Y is None:
        d = np.diagonal(K)
        outer = np.outer(d, d)
    else:
        outer = np.outer(np.sum(dy, axis=0), np.sum(dx, axis=0))
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.nan_to_num(np.divide(K, np.sqrt(outer)))


def level_counts(params, n_iter, X, row):
    """tv [len(X), n_iter + 1, k + 1] of row `row` of fit_transform(X), per level."""
    sm, levels = _levels(params, n_iter, X, None)
    return np.array([[[float(t) for t in sm_oracle.counts(gx[row], gx[c], sm.kv, sm.ke, sm.k)] for gx, _ in levels]
                     for c in range(len(X))])
