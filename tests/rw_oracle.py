"""NumPy restatement of the random walk kernels' per-pair values (random_walk.py:249-341, 468-541) in the form the
device evaluates them: conjugate gradients with the iteration count, the power series by matvecs, the spectral pair
sums.  Graphs are (A, labels or None) with A the reference's dense adjacency matrix."""
import numpy as np


def cg_matvec(Ax, Ay, Lx=None, Ly=None):
    """M p of the conjugate-gradient operator: Ax P Ay (P = p in Fortran order), each label pair (a, b) taking
    Ax[u, v] with L(u) = a, L(v) = b and Ay[v', u'] with L'(v') = a, L'(u') = b."""
    xs, ys = Ax.shape[0], Ay.shape[0]
    if Lx is None:
        return lambda p: (Ax @ p.reshape((xs, ys), order="F") @ Ay).reshape(-1, order="F")
    Lx, Ly = np.asarray(Lx), np.asarray(Ly)
    common = set(Lx.tolist()) & set(Ly.tolist())
    pairs = [(a, b) for a in common for b in common]
    mats = [(Ax * np.outer(Lx == a, Lx == b), Ay * np.outer(Ly == a, Ly == b)) for a, b in pairs]

    def mv(p):
        P = p.reshape((xs, ys), order="F")
        y = np.zeros((xs, ys))
        for X, Y in mats:
            y += X @ P @ Y
        return y.reshape(-1, order="F")
    return mv


def cg_pair(Ax, Ay, lamda, Lx=None, Ly=None, rtol=1e-6, maxiter=20):
    """(sum(x), iterations) of scipy's cg on (I - lamda M) x = 1 from x0 = 0."""
    mn = Ax.shape[0] * Ay.shape[0]
    if mn == 0:
        return 0.0, 0
    mv = cg_matvec(Ax, Ay, Lx, Ly)
    b = np.ones(mn)
    atol = rtol * np.linalg.norm(b)
    x, r = np.zeros(mn), b.copy()
    p = None
    rho_prev = None
    for it in range(maxiter):
        if np.linalg.norm(r) < atol:
            return float(np.sum(x)), it
        rho = np.dot(r, r)
        p = r.copy() if it == 0 else p * (rho / rho_prev) + r
        q = p - lamda * mv(p)
        alpha = rho / np.dot(p, q)
        x += alpha * p
        r -= alpha * q
        rho_prev = rho
    return float(np.sum(x)), maxiter


def product_matrix(Ax, Ay, Lx=None, Ly=None):
    """sum over common label pairs of kron(Ax^ab, Ay^ab) = D kron(Ax, Ay) D."""
    M = np.kron(Ax, Ay)
    if Lx is not None:
        d = (np.asarray(Lx)[:, None] == np.asarray(Ly)[None, :]).reshape(-1)
        M = M * np.outer(d, d)
    return M


def series_pair(Ax, Ay, coef, Lx=None, Ly=None):
    """sum_k coef[k] 1^T M^k 1 and the sum of the terms' magnitudes."""
    M = product_matrix(Ax, Ay, Lx, Ly)
    v = np.ones(M.shape[0])
    S, mag = coef[0] * v.sum(), abs(coef[0] * v.sum())
    for c in coef[1:]:
        v = M @ v
        S += c * v.sum()
        mag += abs(c * v.sum())
    return S, mag


def expm_pair(Ax, Ay, lamda, Lx=None, Ly=None):
    from scipy.linalg import expm
    return float(np.sum(expm(lamda * product_matrix(Ax, Ay, Lx, Ly))))


def spectral_pair(qx, wx, qy, wy, f):
    """sum_ab (q_a q'_b)^2 f(w_a w'_b) and the sum of the terms' magnitudes."""
    ff = np.kron(qx, qy)
    t = ff * ff * f(np.kron(wx, wy))
    return float(np.sum(t)), float(np.sum(np.abs(t)))


def eig_data(A):
    """(real(1^T V), real(w)) of numpy.linalg.eig, the reference's `sd`."""
    w, v = np.linalg.eig(A)
    return np.real(np.sum(v, axis=0)), np.real(w)
