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


def cg_trace(Ax, Ay, lamda, Lx=None, Ly=None, rtol=1e-6, maxiter=20, iters=None):
    """(sum(x), iterations, [||r|| at each norm test], atol) of scipy's cg on (I - lamda M) x = 1 from x0 = 0.
    `iters`: run exactly that many iterations, whatever the norm tests say."""
    mn = Ax.shape[0] * Ay.shape[0]
    if mn == 0:
        return 0.0, 0, [], 0.0
    mv = cg_matvec(Ax, Ay, Lx, Ly)
    b = np.ones(mn)
    atol = rtol * np.linalg.norm(b)
    x, r = np.zeros(mn), b.copy()
    p = None
    rho_prev = None
    norms = []
    for it in range(maxiter if iters is None else iters):
        norms.append(np.linalg.norm(r))
        if iters is None and norms[-1] < atol:
            return float(np.sum(x)), it, norms, atol
        rho = np.dot(r, r)
        p = r.copy() if it == 0 else p * (rho / rho_prev) + r
        q = p - lamda * mv(p)
        alpha = rho / np.dot(p, q)
        x += alpha * p
        r -= alpha * q
        rho_prev = rho
    norms.append(np.linalg.norm(r))
    return float(np.sum(x)), maxiter if iters is None else iters, norms, atol


def cg_pair(Ax, Ay, lamda, Lx=None, Ly=None, rtol=1e-6, maxiter=20):
    """(sum(x), iterations) of scipy's cg on (I - lamda M) x = 1 from x0 = 0."""
    return cg_trace(Ax, Ay, lamda, Lx, Ly, rtol, maxiter)[:2]


def product_matrix(Ax, Ay, Lx=None, Ly=None):
    """sum over common label pairs of kron(Ax^ab, Ay^ab) = D kron(Ax, Ay) D."""
    M = np.kron(Ax, Ay)
    if Lx is not None:
        d = (np.asarray(Lx)[:, None] == np.asarray(Ly)[None, :]).reshape(-1)
        M = M * np.outer(d, d)
    return M


def series_pair(Ax, Ay, coef, Lx=None, Ly=None):
    """sum_k coef[k] 1^T M^k 1 and the sum of the terms' magnitudes."""
    M = sparse_product_matrix(Ax, Ay, Lx, Ly)
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


def sparse_product_matrix(Ax, Ay, Lx=None, Ly=None):
    """product_matrix as a scipy.sparse CSR matrix."""
    import scipy.sparse as sp
    M = sp.kron(sp.csr_matrix(Ax), sp.csr_matrix(Ay), format="csr")
    if Lx is not None:
        d = sp.diags((np.asarray(Lx)[:, None] == np.asarray(Ly)[None, :]).reshape(-1).astype(float))
        M = (d @ M @ d).tocsr()
    return M


def taylor_pair(Ax, Ay, lamda, Lx=None, Ly=None):
    """sum_k lamda^k / k! 1^T M^k 1 = 1^T expm(lamda M) 1 for non-negative A, summed to convergence with sparse
    matvecs on the scaled terms v_k = lamda^k / k! M^k 1 (which stay finite where M^k 1 overflows).  Stops once the
    terms decrease geometrically (k >= 2 lamda R_i R_j, R the largest row sum) and are below 2^-60 of the sum."""
    M = sparse_product_matrix(Ax, Ay, Lx, Ly)
    n = M.shape[0]
    if n == 0:
        return 0.0
    kmin = 2.0 * lamda * np.max(np.sum(Ax, axis=1), initial=0.0) * np.max(np.sum(Ay, axis=1), initial=0.0)
    v = np.ones(n)
    S = float(n)
    k = 0
    while True:
        k += 1
        v = (lamda / k) * (M @ v)
        t = float(v.sum())
        S += t
        if t == 0.0 or (k >= kmin and t < 2.0 ** -60 * S):
            return S


def device_taylor(Ax, Ay, lamda, scaled, cap=2000):
    """(sum, terms, cap reached) of the device's Taylor series for unlabelled graphs, operation for operation:
    `scaled` False replays s_k = M^k 1 with c_k = lamda^k / k! kept apart (term c_k 1^T s_k), True the scaled vector
    s_k = (lamda / k) M s_{k-1} (term 1^T s_k); the stopping rule is the device's (k >= 2 lamda R_i R_j and the term
    below 2^-56 of the sum, or a zero vector sum, at most `cap` terms)."""
    M = sparse_product_matrix(Ax, Ay)
    kmin = 2.0 * lamda * np.max(np.sum(Ax, axis=1)) * np.max(np.sum(Ay, axis=1))
    s = np.ones(M.shape[0])
    c, S = 1.0, float(M.shape[0])
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        for k in range(1, cap + 1):
            if scaled:
                s = (lamda / k) * (M @ s)
                term = s.sum()
            else:
                s = M @ s
                c = c * lamda / k
                term = c * s.sum()
            S += term
            if k >= kmin and abs(term) < 2.0 ** -56 * abs(S):
                return S, k, False
            if s.sum() == 0.0:
                return S, k, False
    return S, cap, True


def hub_graphs():
    """{name: adjacency} of graphs whose Taylor series overflows M^k 1 before its stopping bound at lamda = 0.1 (a
    complete graph K31, a 60-vertex path with one vertex joined to 40 of the others, a star of 100 leaves) and the
    complete graph K21, where it does not."""
    def complete(n):
        return np.ones((n, n)) - np.eye(n)
    hub = np.zeros((60, 60))
    hub[0, 1:41] = 1
    hub[np.arange(1, 59), np.arange(2, 60)] = 1
    star = np.zeros((101, 101))
    star[0, 1:] = 1
    return {"K21": complete(21), "K31": complete(31), "hub60": hub + hub.T, "star100": star + star.T}


def symmetric_expm_pair(Ax, Ay, lamda):
    """1^T expm(lamda kron(Ax, Ay)) 1 for symmetric A from eigh: sum_ab (q_a q'_b)^2 exp(lamda w_a w'_b), every term
    non-negative.  Stands in for expm_pair where kron(Ax, Ay) is too large for a dense expm."""
    wx, vx = np.linalg.eigh(Ax)
    wy, vy = np.linalg.eigh(Ay)
    return spectral_pair(vx.sum(0), wx, vy.sum(0), wy, lambda z: np.exp(lamda * z))[0]


def spectral_pair(qx, wx, qy, wy, f):
    """sum_ab (q_a q'_b)^2 f(w_a w'_b) and the sum of the terms' magnitudes."""
    ff = np.kron(qx, qy)
    t = ff * ff * f(np.kron(wx, wy))
    return float(np.sum(t)), float(np.sum(np.abs(t)))


def eig_data(A):
    """(real(1^T V), real(w)) of numpy.linalg.eig, the reference's `sd`."""
    w, v = np.linalg.eig(A)
    return np.real(np.sum(v, axis=0)), np.real(w)
