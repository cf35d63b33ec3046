"""CPU oracle of SubgraphMatching (test infrastructure): the definition restated in Python / NumPy.

For graphs x, y (as SubgraphMatching.parse_input returns them: n, edges, vertex labels, edge labels) the weighted
product graph has the vertices p = (a, b), in lexicographic order, with cv = kv(La, Lb) != 0.  Between p and q that
share no vertex, with h the one of larger x vertex and l the other, ce is -1 when neither h.a -> l.a nor h.b -> l.b is
an edge, 0 when one of them is, and ke of their labels (1 for ke=None) when both are.  tv[s - 1] sums
prod cv * prod |ce| over the vertex sets of size s that are cliques of ce != 0 and connected by the ce > 0 edges.

The sets are enumerated from their smallest vertex, growing connected sets by c-neighbours: a set S with extension
candidates C takes each candidate w in turn; the child's candidates are the remaining ones adjacent to w plus the
c-neighbours of w above the root that have a d-edge to every vertex of S.  The terms are kept as exact fractions
when `exact`, so the result does not depend on the summation order."""
from fractions import Fraction

import numpy as np


def product_graph(x, y, kv, ke):
    """(cv [nv], ce [nv, nv], vertex pairs [nv, 2]) of the weighted product graph."""
    nx, ex, lx, elx = x
    ny, ey, ly, ely = y
    Ex = {e: (elx[i] if elx is not None else None) for i, e in enumerate(ex)}
    Ey = {e: (ely[i] if ely is not None else None) for i, e in enumerate(ey)}
    V, cv = [], []
    for a in range(nx):
        for b in range(ny):
            c = 1.0 if kv is None else float(kv(lx[a], ly[b]))
            if c != 0.0:
                V.append((a, b))
                cv.append(c)
    nv = len(V)
    ce = np.zeros((nv, nv))
    for s in range(nv):
        for t in range(s):
            (pa, pb), (qa, qb) = V[s], V[t]
            if pa == qa or pb == qb:
                continue
            if pa < qa:
                pa, pb, qa, qb = qa, qb, pa, pb
            ea, eb = (pa, qa) in Ex, (pb, qb) in Ey
            if not ea and not eb:
                w = -1.0
            elif ea != eb:
                w = 0.0
            else:
                w = 1.0 if ke is None else float(ke(Ex[(pa, qa)], Ey[(pb, qb)]))
            ce[s, t] = ce[t, s] = w
    return np.array(cv), ce, V


def counts(x, y, kv, ke, k, exact=True, absolute=False):
    """tv [k + 1] (Fractions when exact; with `absolute`, the sums of |term|)."""
    cv, ce, _ = product_graph(x, y, kv, ke)
    nv = len(cv)
    kk = max(k, 1)
    zero = Fraction(0) if exact else 0.0
    tv = [zero] * (k + 1)
    conv = (lambda v: Fraction(v)) if exact else float
    fix = abs if absolute else (lambda v: v)
    cnb = [np.flatnonzero(ce[v] > 0) for v in range(nv)]

    def grow(S, term, cand, root):
        for i, w in enumerate(cand):
            t = term * conv(cv[w])
            for s in S:
                t *= conv(abs(ce[w, s]))
            tv[len(S)] += fix(t)
            if len(S) + 1 >= kk:
                continue
            nxt = [u for u in cand[i + 1:] if ce[u, w] != 0]
            nxt += [int(u) for u in cnb[w] if u > root and all(ce[u, s] < 0 for s in S)]
            grow(S + [w], t, nxt, root)

    for v in range(nv):
        tv[0] += fix(conv(cv[v]))
        if kk > 1:
            grow([v], conv(cv[v]), [int(u) for u in cnb[v] if u > v], v)
    return tv


def fma_fold(lambdas, tv):
    """sum_s lambda_s tv_s as one chain of correctly rounded fused multiply-adds from 0 (np.dot's order)."""
    acc = 0.0
    for l, t in zip(lambdas, tv):
        acc = float(Fraction(float(l)) * Fraction(float(t)) + Fraction(acc))
    return acc


def sm_value(x, y, kv, ke, k, lambdas):
    tv = counts(x, y, kv, ke, k)
    return fma_fold(np.ravel(lambdas), [float(t) for t in tv])


def gram(X, Y, kv, ke, k, lambdas, normalize=False):
    """The reference's fit_transform (Y None) or transform matrix: K[j, i] = sm(X[j], X[i]) for j <= i, mirrored;
    K[j, i] = sm(Y[j], X[i]); normalised by sqrt(outer(diag(Y), diag(X)))."""
    f = lambda a, b: sm_value(a, b, kv, ke, k, lambdas)
    n = len(X)
    if Y is None:
        K = np.zeros((n, n))
        for i in range(n):
            for j in range(i + 1):
                K[j, i] = K[i, j] = f(X[j], X[i])
        if normalize:
            d = np.diagonal(K).copy()
            with np.errstate(invalid="ignore", divide="ignore"):
                K = K / np.sqrt(np.outer(d, d))
        return K
    K = np.array([[f(y, x) for x in X] for y in Y]).reshape(len(Y), n)
    if normalize:
        dx = np.array([f(x, x) for x in X])
        dy = np.array([f(y, y) for y in Y])
        with np.errstate(invalid="ignore", divide="ignore"):
            K /= np.sqrt(np.outer(dy, dx))
    return K
