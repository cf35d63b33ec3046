"""NumPy restatement of PyramidMatch (pyramid_match.py:178-285) from given embeddings: the cells, the per-level
histogram intersections and the reference's combine replayed operation for operation (both statements inside the
level loop).  K equals the reference's bit for bit given the same |U|."""
import numpy as np


def split_calls(U, shapes):
    """The golden's padded [rows, d] array and (n, n_cols) list -> one [n, n_cols] array per embedding call."""
    out, a = [], 0
    for n, c in shapes.tolist():
        out.append(U[a:a + n, :c])
        a += n
    return out


def histograms(us, labels, L, d, n_rows):
    """Per graph, per level: the [n_rows, 2^j] histogram (rows label * d + q, or q when labels is None)."""
    H = []
    for g, u in enumerate(us):
        levels = []
        for j in range(L):
            k = 2 ** j
            D = np.zeros((n_rows, k))
            T = np.floor(u * k)
            T[T == k] = k - 1
            for p in range(u.shape[0]):
                for q in range(u.shape[1]):
                    row = q if labels is None else labels[g][p] * d + q
                    D[row, int(T[p, q])] += 1
            levels.append(D)
        H.append(levels)
    return H


def pair(x, y, L):
    k = 0
    if len(x) != 0 and len(y) != 0:
        intersec = np.zeros(L)
        for p, xp, yp in zip(range(L), x, y):
            r = min(xp.shape[0], yp.shape[0])
            intersec[p] = np.sum(np.minimum(xp[:r], yp[:r]))
            k += intersec[L - 1]
            for q in range(L - 1):
                k += (1.0 / (2 ** (L - q - 1))) * (intersec[q] - intersec[q + 1])
    return k


def label_enumeration(fit_labels, tr_labels=None):
    """Label ids: the fit labels first (any order: K does not depend on it), then the transform's unseen ones."""
    known = {}
    for L in fit_labels:
        for l in L:
            known.setdefault(l, len(known))
    n_fit = len(known)
    for L in tr_labels or []:
        for l in L:
            known.setdefault(l, len(known))
    return known, n_fit


def kernel(us_fit, L, d, labels_fit=None, us_tr=None, labels_tr=None, normalize=False):
    """(K_fit_transform, K_transform or None) as the reference computes them."""
    if labels_fit is None:
        rows_fit = rows_all = d
        lf = lt = None
    else:
        known, n_fit = label_enumeration(labels_fit, labels_tr)
        rows_fit, rows_all = n_fit * d, len(known) * d
        lf = [[known[l] for l in Lg] for Lg in labels_fit]
        lt = None if labels_tr is None else [[known[l] for l in Lg] for Lg in labels_tr]
    Hx = histograms(us_fit, lf, L, d, rows_fit)
    n = len(Hx)
    K = np.zeros((n, n))
    for i in range(n):
        for j in range(i, n):
            K[i, j] = pair(Hx[i], Hx[j], L)
    K = np.triu(K) + np.triu(K, 1).T
    xd = np.diagonal(K).copy()
    Kt = None
    if us_tr is not None:
        Hy = histograms(us_tr, lt, L, d, rows_all)
        Kt = np.array([[pair(y, x, L) for x in Hx] for y in Hy]).reshape(len(Hy), n)
        if normalize:
            yd = np.array([pair(y, y, L) for y in Hy], dtype=float)
            with np.errstate(invalid="ignore", divide="ignore"):
                Kt = Kt / np.sqrt(np.outer(yd, xd))
    if normalize:
        with np.errstate(invalid="ignore", divide="ignore"):
            K = K / np.sqrt(np.outer(xd, xd))
    return K, Kt
