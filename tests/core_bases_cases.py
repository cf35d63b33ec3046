"""Inputs of the CoreFramework-over-NeighborhoodHash / OddSth / WL-OA / SubgraphMatching goldens
(tests/golden/core_bases.npz), generated from seeds."""
import numpy as np

BASES = {
    "nh": ("NH", {"random_state": 3}),
    "nhcs": ("NH", {"random_state": 5, "nh_type": "count_sensitive", "R": 2}),
    "nhrs": ("NH", {"random_state": "shared"}),  # one RandomState(11) for every level (params_of)
    "nhgl": ("NH", {"random_state": None}),  # numpy's global stream, seeded with GLOBAL_SEED before every case
    "oddN": ("ODD", {}),
    "odd2": ("ODD", {"h": 2}),
    "wloa": ("WLOA", {"n_iter": 3}),
    "smN": ("SM", {"k": 3, "ke": None}),
    "sm": ("SM", {"k": 3}),
}

GLOBAL_SEED = 13


def params_of(name):
    """A fresh copy of the base's parameters: a "shared" random_state becomes a new RandomState(11), which the levels
    of one estimator then consume in turn."""
    kind, params = BASES[name]
    params = dict(params)
    if params.get("random_state") == "shared":
        params["random_state"] = np.random.RandomState(11)
    return kind, params


def graphs(n, nbar, seed, new_labels=False, dense=0.0, isolated=False):
    """[edge dictionary {(u, v): 1}, vertex labels, edge labels] of undirected random graphs.  `dense` adds a clique
    over the first vertices of some graphs, so that their maximum core is higher; `isolated` appends a graph that is
    one vertex without an edge (as an adjacency matrix)."""
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
        if dense and rs.rand() < dense:
            c = min(k, 6)
            for a in range(c):
                for b in range(c):
                    if a != b:
                        g[(a, b)] = 1
        for v in range(k):  # every vertex sits on an edge
            if not any(a == v for a, _ in g):
                w = (v + 1) % k
                g[(v, w)] = 1
                g[(w, v)] = 1
        E = {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}
        out.append([g, L, E])
    if isolated:
        out.append([np.zeros((1, 1)), {0: 1}, {}])
    return out


def fit_set():
    return graphs(10, 10, 7)


def transform_set():
    """New labels, and graphs whose maximum core exceeds the fitted one's."""
    return graphs(5, 10, 8, new_labels=True, dense=0.6)


def isolated_set():
    return graphs(4, 8, 9, isolated=True)


def unlabelled_edges_set():
    """The fit set without edge labels."""
    return [[g, L] for g, L, _ in fit_set()]
