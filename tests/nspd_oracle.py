"""NumPy / Python restatement of NeighborhoodSubgraphPairwiseDistance (neighborhood_subgraph_pairwise_distance.py),
written from its definition for the tests: the graphs come from the package's own parser (`_nspd_graph`: indices of
the sorted symbols, edges with a positive adjacency entry), the neighbourhoods and distances follow graph.py's
produce_neighborhoods (ball l + 1 is the union of the level-l balls over the level-l ball), the sub-edge sets are real
Python sets (so their order is the running interpreter's) and APHash is restated below.  K follows the reference's
numpy semantics: int64 Grams and diagonal products, float64 sqrt and division, nan_to_num."""
import numpy as np

from grakel_b200.kernels import _nspd_graph


def aphash(word):
    """Arash Partow's hash over the first len(word) bytes of the UTF-8 encoding, bytes as signed char."""
    bs = word.encode("utf-8")
    h = 0xAAAAAAAA
    for i in range(len(word)):
        c = bs[i] - 256 if bs[i] >= 128 else bs[i]
        c &= 0xFFFFFFFF
        if i & 1 == 0:
            h ^= ((h << 7) & 0xFFFFFFFF) ^ ((c * (h >> 3)) & 0xFFFFFFFF)
        else:
            h ^= (~((((h << 11) & 0xFFFFFFFF) + (c ^ (h >> 5))) & 0xFFFFFFFF)) & 0xFFFFFFFF
        h &= 0xFFFFFFFF
    return h


def neighborhoods(n, edges, r, d):
    """(N[level][v] as lists, D[delta] as sets of pairs, Dist_pair) as produce_neighborhoods(r, with_distances, d)."""
    out = {i: [] for i in range(n)}
    for i, j in edges:
        out[i].append(j)
    N = {0: {i: {i} for i in range(n)}}
    D = {0: {(i, i) for i in range(n)}}
    dp = {(i, i): 0 for i in range(n)}
    if r > 0:
        N[1] = {}
        if d >= 1:
            D[1] = set()
        for i in range(n):
            N[1][i] = sorted([i] + out[i])
            if d >= 1:
                s = {(i, k) for k in out[i]}
                dp.update(dict.fromkeys(s, 1))
                D[1] |= s
        for level in range(1, max(r, d)):
            N[level + 1] = {}
            if level <= d - 1:
                D[level + 1] = set()
            for i in range(n):
                nb = set()
                for w in N[level][i]:
                    nb |= set(N[level][w])
                N[level + 1][i] = sorted(nb)
                if level <= d - 1:
                    s = {(i, j) for j in nb - set(N[level][i])}
                    dp.update(dict.fromkeys(s, level + 1))
                    D[level + 1] |= s
    return N, D, dp


_HASHES = {}


def hashes(graph, r, d):
    """H[(rho, v)] of one parsed graph (n, edges, vertex label strings, edge label strings), memoised: a test that
    compares fit_transform, transform and their normalised forms hashes every graph once."""
    key = (graph[0], tuple(graph[1]), tuple(graph[2]), tuple(graph[3]), r, d)
    if key not in _HASHES:
        _HASHES[key] = _hashes(graph, r, d)
    return _HASHES[key]


def _hashes(graph, r, d):
    n, edges, vl, el = graph
    elab = dict(zip(edges, el))
    N, D, dp = neighborhoods(n, edges, r, d)
    H = {}
    for v in range(n):
        re = sorted(edges)
        for rho in range(r, -1, -1):
            sub = sorted(N[rho][v])
            re = {(i, j) for (i, j) in re if i in sub and j in sub}
            enc, lab = "", {}
            for i in sub:
                s = "|".join(sorted(str(dp[(i, j)]) + "," + vl[j] for j in sub if (i, j) in dp))
                enc += s + "."
                lab[i] = s
            enc = enc[:-1] + ":"
            for (i, j) in re:
                enc += lab[i] + "," + lab[j] + "," + elab[(i, j)] + "_"
            H[rho, v] = aphash(enc)
    return H, D


def features(graphs, r, d, fit_keys=None):
    """{(rho, delta): int64 count matrix} in first-occurrence order, the per-graph hashes and the key dictionaries."""
    data, keys, Hs = {}, {}, []
    for g, graph in enumerate(graphs):
        H, D = hashes(graph, r, d)
        Hs.append(H)
        for delta in range(d + 1):
            if delta not in D:
                continue
            for (a, b) in D[delta]:
                for rho in range(r + 1):
                    k = keys.setdefault((rho, delta), {})
                    fk = {} if fit_keys is None else fit_keys.get((rho, delta), {})
                    key = (H[rho, a], H[rho, b])
                    idx = fk.get(key)
                    if idx is None:
                        idx = k.setdefault(key, len(k) + len(fk))
                    row = data.setdefault((rho, delta), {})
                    row[g, idx] = row.get((g, idx), 0) + 1
    M = {}
    for lev, entries in data.items():
        width = len(keys[lev]) + (0 if fit_keys is None else len(fit_keys.get(lev, {})))
        m = np.zeros((len(graphs), width), dtype=np.int64)
        for (g, i), c in entries.items():
            m[g, i] = c
        M[lev] = m
    return M, Hs, keys


def parse(X):
    return [_nspd_graph(*x) for x in X]


def fit_transform(X, r=3, d=4, normalize=False):
    M, _, _ = features(parse(X), r, d)
    S = np.zeros((len(X), len(X)))
    for m in M.values():
        K = m @ m.T
        kd = K.diagonal()
        with np.errstate(invalid="ignore", divide="ignore"):
            Q = K / np.sqrt(np.outer(kd, kd))
        np.fill_diagonal(Q, np.nan_to_num(np.diag(Q), nan=1.0))
        S = S + np.nan_to_num(Q)
    return S / len(M) if normalize else S


def transform(X, Y, r=3, d=4, normalize=False):
    MX, _, keys = features(parse(X), r, d)
    MY, _, _ = features(parse(Y), r, d, fit_keys=keys)
    S = np.zeros((len(Y), len(X)))
    for lev, my in MY.items():
        if lev not in MX:
            continue
        mx = MX[lev]
        K = (mx @ my[:, :mx.shape[1]].T).T
        with np.errstate(invalid="ignore", divide="ignore"):
            S += np.nan_to_num(K / np.sqrt(np.outer((my ** 2).sum(-1), (mx ** 2).sum(-1))))
    if normalize:
        S /= np.sqrt(np.outer(np.full(len(Y), float(len(MY))), np.full(len(X), float(len(MX)))))
    return S


def vertex_hashes(X, r=3, d=4):
    """[r + 1, total vertices] uint32: H[rho, v] of every graph's vertices, graph after graph."""
    out = []
    for graph in parse(X):
        H, _ = hashes(graph, r, d)
        out.append(np.array([[H[rho, v] for v in range(graph[0])] for rho in range(r + 1)], dtype=np.uint32)
                   .reshape(r + 1, graph[0]))
    return np.concatenate(out, axis=1)
