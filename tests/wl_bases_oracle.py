"""CPU restatement of WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance / OddSth (weisfeiler_lehman.py:
160-270, 366-482): the joint WL partition of the fitted and transformed graphs (oracle.gk_oracle), numbered as the
reference numbers it (wl_reference_dictionaries), then the base kernel's restatement (nspd_oracle / odd_oracle) on
every level's labels, the levels' K summed in level order as np.sum(axis=0) does."""
import numpy as np

import nspd_oracle
import odd_oracle
from grakel_b200.kernels import wl_reference_dictionaries
from grakel_b200.packing import label_ids, pack
from oracle.gk_oracle import WLOracle, wl_partitions


def level_elements(X, Y, n_iter):
    """Every level's elements [edges, {vertex: reference label}, edge labels] of X and of Y (None without Y)."""
    XY = list(X) + list(Y or [])
    block = pack(XY, "wl", len_ok=lambda n: n >= 2)
    bx = pack(list(X), "wl", len_ok=lambda n: n >= 2)
    ids_x, d0 = label_ids(bx.labels, None, sort_new=True)
    ids = ids_x
    if Y:
        by = pack(list(Y), "wl", len_ok=lambda n: n >= 2)
        ids_y, _ = label_ids(by.labels, d0, sort_new=True)
        ids = np.concatenate([ids_x, ids_y])
    _, levels = WLOracle(n_iter=n_iter).fit_transform(XY, return_levels=True)
    _, labels = wl_reference_dictionaries(np.asarray(block.row_ptr), np.asarray(block.col_idx), ids, len(d0),
                                          wl_partitions(levels), n_fit_vertices=bx.n_vertices)
    gp = np.asarray(block.graph_ptr)
    out = []
    for lab in labels:
        els = [[x[0], {k: int(lab[gp[j] + i]) for i, k in enumerate(x[1].keys())}] + list(x[2:])
               for j, x in enumerate(XY)]
        out.append((els[:len(X)], els[len(X):] if Y else None))
    return out


def kernel(kind, params, n_iter, X, Y=None):
    """Un-normalised K of fit_transform(X), or of transform(Y) after fit(X)."""
    Ks = []
    for lx, ly in level_elements(X, Y, n_iter):
        if kind == "NSPD":
            r, d = params.get("r", 3), params.get("d", 4)
            Ks.append(nspd_oracle.fit_transform(lx, r, d) if ly is None else nspd_oracle.transform(lx, ly, r, d))
        else:
            Ks.append(odd_oracle.kernel(lx, ly, h=params.get("h")))
    return np.sum(Ks, axis=0)


def normalized(K):
    d = np.diagonal(K)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.nan_to_num(np.divide(K, np.sqrt(np.outer(d, d))))
