"""Inputs of the WeisfeilerLehman-over-NSPD / OddSth goldens (tests/golden/wl_bases.npz), generated from seeds."""
import numpy as np

BASES = {
    "nspd00": ("NSPD", {"r": 0, "d": 0}),
    "nspd12": ("NSPD", {"r": 1, "d": 2}),
    "nspd34": ("NSPD", {"r": 3, "d": 4}),
    "oddN": ("ODD", {}),
    "odd2": ("ODD", {"h": 2}),
}
N_ITERS = (1, 2, 5)


def graphs(n, nbar, seed, new_labels=False):
    """[edge dictionary, vertex labels, edge labels] of undirected random graphs; with `new_labels` some vertices carry
    labels the fitted graphs never have (7 and 8)."""
    rs = np.random.RandomState(seed)
    out = []
    for _ in range(n):
        k = int(rs.randint(nbar // 2, nbar + nbar // 2 + 1))
        p = 3.0 / max(k - 1, 1)
        iu = np.triu_indices(k, 1)
        m = rs.rand(len(iu[0])) < p
        L = {i: int(rs.randint(9 if new_labels else 7)) for i in range(k)}
        g = {}
        for a, b in zip(iu[0][m].tolist(), iu[1][m].tolist()):
            g[(a, b)] = 1
            g[(b, a)] = 1
        for v in range(k):  # every vertex sits on an edge, so the base kernels see all WL vertices
            if not any(a == v for a, _ in g):
                w = (v + 1) % k
                g[(v, w)] = 1
                g[(w, v)] = 1
        E = {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}
        out.append([g, L, E])
    return out


def fit_set():
    return graphs(10, 10, 7)


def transform_set():
    return graphs(4, 10, 8, new_labels=True)
