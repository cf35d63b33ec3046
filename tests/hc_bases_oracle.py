"""CPU restatement of HadamardCode over SubgraphMatching and NeighborhoodSubgraphPairwiseDistance (hadamard_code.py
:134-257): every level's Hadamard-code vectors from tests/hc_oracle.py (the fitted graphs at the fit enumeration's
width, the transformed ones at the extended enumeration's width), every level's elements [graph, {vertex: tuple of
numpy int64}, edge labels] handed to the base kernel's restatement (tests/sm_oracle.py, tests/nspd_oracle.py), and the
levels summed in level order as np.sum(axis=0) does."""
import numpy as np

import hc_oracle
import nspd_oracle
import sm_oracle
from grakel_b200 import SubgraphMatching


def level_elements(X, n_iter, enum):
    """Per level, the elements the reference hands its base kernel at that level."""
    out = []
    for level in hc_oracle.levels(X, n_iter, enum):
        out.append([[x[0], {k: tuple(v) for k, v in d.items()}] + list(x[2:3]) for x, d in zip(X, level)])
    return out


def _levels(X, Y, n_iter):
    ex = hc_oracle.enumerate_labels([x[1] for x in X])
    lx = level_elements(X, n_iter, ex)
    if Y is None:
        return [(a, None) for a in lx]
    ey = hc_oracle.enumerate_labels([y[1] for y in Y], ex)
    return list(zip(lx, level_elements(Y, n_iter, ey)))


def sm_kernel(params, n_iter, X, Y=None, normalize=False):
    """K of fit_transform(X), or of transform(Y) after fit(X)."""
    sm = SubgraphMatching(**params)
    sm.initialize()
    Ks, dx, dy = [], [], []
    for lx, ly in _levels(X, Y, n_iter):
        gx = sm.parse_input(lx)
        gy = None if ly is None else sm.parse_input(ly)
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


def nspd_kernel(params, n_iter, X, Y=None):
    """Un-normalised K of fit_transform(X), or of transform(Y) after fit(X)."""
    r, d = params.get("r", 3), params.get("d", 4)
    Ks = []
    for lx, ly in _levels(X, Y, n_iter):
        Ks.append(nspd_oracle.fit_transform(lx, r, d) if ly is None else nspd_oracle.transform(lx, ly, r, d))
    return np.sum(Ks, axis=0)
