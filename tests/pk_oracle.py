"""NumPy restatement of Propagation / PropagationAttr (propagation.py:249-423, 585-689): the reference's per-level
hashes with its numpy operations, and K from the bins by (graph, bin) counts.  Test infrastructure only."""
import numpy as np


def levels(Ts, sizes, P, us, bs, w, sqrt=False, attr=False, dim_orig=None, labels=None):
    """Per level (bins, private flags) of one side's vertices.  P: the initial V x D matrix in its dtype (one-hot
    float64 for labels).  dim_orig / labels: a transform with labels unseen at fit (labels >= dim_orig are new)."""
    idx = np.concatenate([[0], np.cumsum(sizes)])
    P = P.copy()
    V = P.shape[0]
    split = dim_orig is not None and dim_orig < P.shape[1]
    priv = (np.asarray(labels) >= dim_orig) if split else np.zeros(V, dtype=bool)
    out = []
    for t in range(len(us)):
        if attr:
            bins = np.floor((P * us[t] + bs[t]) / w)
        else:
            X = np.sqrt(P) if sqrt else P
            bins = np.empty(V)
            if split:
                bins[~priv] = np.floor((np.dot(X[~priv][:, :dim_orig], us[t][:dim_orig]) + bs[t]) / w)
                bins[priv] = np.floor((np.dot(X[priv], us[t]) + bs[t]) / w)
            else:
                bins = np.floor((np.dot(X, us[t]) + bs[t]) / w)
        out.append((bins, priv.copy()))
        if t < len(us) - 1:
            for k in range(len(sizes)):
                a, b = idx[k], idx[k + 1]
                P[a:b, :] = np.dot(Ts[k], P[a:b, :])
            if split:
                priv = np.all(P[:, dim_orig:] > 0, axis=1)
    return out


def counts(lv, sizes, split=False):
    """Per level: list of {key: count} per graph; key = (private, bin tuple).  `split` counts a vertex also in every
    earlier graph k with idx[k + 1] == v (the reference's inclusive bound)."""
    idx = np.concatenate([[0], np.cumsum(sizes)])
    out = []
    for bins, priv in lv:
        b2 = bins.reshape(len(bins), -1) + 0.0  # -0.0 -> 0.0
        per = []
        for k in range(len(sizes)):
            hi = idx[k + 1] + 1 if split else idx[k + 1]
            c = {}
            for v in range(idx[k], min(hi, len(b2))):
                key = (bool(priv[v]), tuple(b2[v].tolist()))
                c[key] = c.get(key, 0) + 1
            per.append(c)
        out.append(per)
    return out


def gram(cx, cy=None):
    """K = sum over levels of the (graph, bin) count dot products; private bins of Y never match X."""
    cy = cx if cy is None else cy
    K = np.zeros((len(cy[0]), len(cx[0])))
    for lx, ly in zip(cx, cy):
        for i, a in enumerate(ly):
            for j, b in enumerate(lx):
                K[i, j] += sum(n * b.get(key, 0) for key, n in a.items() if not key[0])
    return K


def diag(c):
    return np.array([sum(sum(n * n for n in g.values()) for g in (lv[k] for lv in c)) for k in range(len(c[0]))],
                    dtype=float)
