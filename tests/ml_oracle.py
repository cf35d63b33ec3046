"""A numpy restatement of MultiscaleLaplacian (multiscale_laplacian.py) with Cholesky factorisations in place of the
reference's inv / eigvals: the CPU arm the device is checked against.  Test infrastructure only.

`els` is a list of (A, phi): symmetric adjacency with non-negative weights and the attribute matrix."""
import numpy as np

POS = 1e-6


def laplacian(A):
    """scipy.sparse.csgraph.laplacian of a dense matrix: the diagonal ignored, degrees from column sums."""
    B = np.array(A, dtype=float)
    np.fill_diagonal(B, 0.0)
    return np.diag(B.sum(axis=0)) - B


def neighbourhoods(A, L):
    """Level l = 1 .. L: the reference's produce_neighborhoods(r=L, sort_neighbors=False) lists ([v] + neighbours at
    level 1, sets after).  Level l + 1 unites the level-l lists of the level-l neighbours: radius 2^(l-1)."""
    n = A.shape[0]
    N = {1: {i: [i] + np.nonzero(A[i] > 0)[0].tolist() for i in range(n)}}
    for l in range(1, L):
        N[l + 1] = {i: sorted(set().union(*[set(N[l][w]) for w in N[l][i]])) for i in range(n)}
    return N


def record(Lap, U, gamma):
    """(S^-1, log det S) of S = U^T Lap^-1 U + gamma I, by Cholesky."""
    R = np.linalg.cholesky(Lap)
    Y = np.linalg.solve(R, U)
    S = Y.T @ Y + gamma * np.eye(U.shape[1])
    T = np.linalg.cholesky(S)
    Z = np.linalg.inv(T)
    return Z.T @ Z, 2.0 * np.sum(np.log(np.diag(T)))


def flg(x, y):
    T = np.linalg.cholesky(x[0] + y[0])
    logr = (-2.0 * np.sum(np.log(np.diag(T))) - 0.5 * (x[1] + y[1])) / 2.0
    return 0.0 if logr < -30 else float(np.exp(logr))


def flg_many(xs, ys):
    """flg over pairs (xs[i], ys[i]), batched."""
    M = np.stack([x[0] + y[0] for x, y in zip(xs, ys)])
    T = np.linalg.cholesky(M)
    ld = 2.0 * np.sum(np.log(np.diagonal(T, axis1=1, axis2=2)), axis=1)
    logr = (-ld - 0.5 * (np.array([x[1] for x in xs]) + np.array([y[1] for y in ys]))) / 2.0
    return np.where(logr < -30, 0.0, np.exp(logr))


def flg_matrix(rows, cols):
    """[flg(r, c) for c in cols] for r in rows."""
    if not rows or not cols:
        return np.zeros((len(rows), len(cols)))
    xs = [r for r in rows for _ in cols]
    ys = [c for _ in rows for c in cols]
    return flg_many(xs, ys).reshape(len(rows), len(cols))


def truncate(K, P, eig=np.linalg.eig):
    v, w = eig(K)
    v, w = np.real(v), np.real(w.T)
    vpos = np.argpartition(v, -P)[-P:]
    vpos = vpos[np.where(v[vpos] > POS)]
    return v[vpos], w[vpos]


class MLOracle:
    def __init__(self, L=3, P=10, gamma=0.01, heta=0.01, n_samples=50, random_state=None, eig=np.linalg.eig):
        self.L, self.P, self.gamma, self.heta, self.n_samples = L, P, gamma, heta, n_samples
        self.rs = np.random.RandomState(random_state) if not isinstance(random_state, np.random.RandomState) \
            else random_state
        self.eig = eig

    def _C(self, A, U, nb):
        Lap = laplacian(A[np.ix_(nb, nb)]) + self.heta * np.eye(len(nb))
        return record(Lap, U[nb, :], self.gamma)

    def _final(self, els, feats):
        return [record(laplacian(A) + self.heta * np.eye(A.shape[0]), F, self.gamma) for (A, _), F in zip(els, feats)]

    def fit(self, els):
        ng = len(els)
        nbs = [neighbourhoods(A, self.L) for A, _ in els]
        V = [(k, j) for k in range(ng) for j in range(els[k][0].shape[0])]
        ns = min(len(V), self.n_samples)
        self.rs.shuffle(V)
        vs = V[:ns]
        self.samples, self.eigs = [list(vs)], []
        phi_k = np.array([els[k][1][j, :] for (k, j) in vs], dtype=float)
        v, w = truncate(phi_k.dot(phi_k.T), self.P, self.eig)
        self.eigs.append((v, w))
        self.ksi = w.dot(phi_k).T / np.sqrt(v)
        feats = [np.asarray(phi, dtype=float).dot(self.ksi) for _, phi in els]
        self.levels = []
        for l in range(1, self.L + 1):
            self.rs.shuffle(V)
            vs = V[:ns]
            self.samples.append(list(vs))
            C = [[self._C(els[k][0], feats[k], nbs[k][l][j]) for j in range(els[k][0].shape[0])] for k in range(ng)]
            Cs = [C[k][j] for (k, j) in vs]
            Kp = [flg_matrix(C[k], Cs) for k in range(ng)]
            K = flg_matrix(Cs, Cs)
            v, w = truncate(K, self.P, self.eig)
            self.eigs.append((v, w))
            Q = w.T / np.sqrt(v)
            feats = [kp.dot(Q) for kp in Kp]
            self.levels.append((Cs, Q))
        self.X = self._final(els, feats)
        return self

    def transform_records(self, els):
        nbs = [neighbourhoods(A, self.L) for A, _ in els]
        feats = [np.asarray(phi, dtype=float).dot(self.ksi) for _, phi in els]
        for l, (Cs, Q) in enumerate(self.levels, start=1):
            nf = []
            for k, (A, _) in enumerate(els):
                Kp = flg_matrix([self._C(A, feats[k], nbs[k][l][j]) for j in range(A.shape[0])], Cs)
                nf.append(Kp.dot(Q))
            feats = nf
        return self._final(els, feats)

    def fit_transform(self, els, normalize=False):
        self.fit(els)
        K = flg_matrix(self.X, self.X)
        if normalize:
            d = np.diagonal(K)
            K = K / np.sqrt(np.outer(d, d))
        return K

    def transform(self, els, normalize=False):
        Y = self.transform_records(els)
        K = flg_matrix(Y, self.X)
        if normalize:
            dx = np.array([flg(x, x) for x in self.X])
            dy = np.array([flg(y, y) for y in Y])
            K = K / np.sqrt(np.outer(dy, dx))
        return K
