"""CPU oracle of SvmTheta (svm_theta.py of the reference): scipy's eigvalsh for the smallest eigenvalue, sklearn's
OneClassSVM for the alphas, the estimator's RandomState for the draws and numpy for the level sums, the means and the
Gram.  It also restates numpy's summation order (`add_reduce`), which the device follows to make phi bit-identical."""
import numpy as np
from scipy.linalg import eigvalsh
from scipy.special import binom
from sklearn.svm import OneClassSVM


def theta_matrix(A):
    """(m, K): the smallest eigenvalue of the 0/1 matrix (upper triangle mirrored) and the matrix the SVM is fit on."""
    K = (np.asarray(A) > 1e-10).astype(float)
    np.fill_diagonal(K, 0.0)
    m = eigvalsh(K, lower=False, subset_by_index=(0, 0))[0]
    if m < 0 and abs(m) > 1e-6:
        K /= -m
        K[np.diag_indices_from(K)] += 1.0
    return m, K


def theta_alphas(A):
    """(m, alphas, n_iter) of one graph."""
    m, K = theta_matrix(A)
    svm = OneClassSVM(kernel="precomputed").fit(K)
    alphas = np.zeros(K.shape[0])
    np.put(alphas, svm.support_, svm._dual_coef_[0])
    return m, alphas, int(np.asarray(svm.n_iter_).reshape(-1)[0])


def distribute(n, subsets_size_range, n_samples):
    """Samples per subset size: floor of each size's binomial share of n_samples, then the leftover samples dealt one
    by one to the sizes from the largest down, wrapping round.  Sizes without a sample are left out; no size at all
    (n below the range) is the reference's ZeroDivisionError."""
    lo, hi = subsets_size_range
    ks = np.arange(lo, min(hi, n) + 1)
    if ks.size == 0:
        raise ZeroDivisionError("no subset size fits the graph")
    c = np.array([binom(n, k) for k in ks], dtype=float)
    base = np.floor(c / c.sum() * n_samples).astype(int)
    for t in range(int(n_samples - base.sum())):
        base[ks.size - 1 - t % ks.size] += 1
    return {int(k): int(v) for k, v in zip(ks, base) if v > 0}


def levels(alphas, subsets_size_range, n_samples, rs, record=None):
    """phi (L, 1) of one graph, drawing from `rs`; `record` collects the drawn index arrays."""
    n = len(alphas)
    lo, hi = subsets_size_range
    samples = distribute(n, subsets_size_range, n_samples)
    phi = np.zeros((hi - lo + 1, 1))
    for i, level in enumerate(range(lo, hi + 1)):
        v = samples.get(level)
        if v is None:
            continue
        sums = []
        for _ in range(v):
            if level <= n:
                idx = rs.choice(n, level, replace=False)
                if record is not None:
                    record.append(idx)
            else:
                idx = range(n)
            sums.append(np.sum(alphas[idx]))
        phi[i] = np.mean(sums)
    return phi


def inner(x, y):
    return np.inner(x, y)[0, 0]


class SvmThetaOracle:
    def __init__(self, random_state=None, n_samples=50, subsets_size_range=(2, 8), metric=inner, normalize=False):
        self.rs = random_state if isinstance(random_state, np.random.RandomState) else \
            np.random.RandomState(random_state)
        self.n_samples, self.range, self.metric, self.normalize = n_samples, subsets_size_range, metric, normalize

    def parse(self, X):
        out = []
        for A in X:
            _, alphas, _ = theta_alphas(A)
            out.append(levels(alphas, self.range, self.n_samples, self.rs))
        return out

    def fit_transform(self, X):
        self.X = self.parse(X)
        n = len(self.X)
        K = np.zeros((n, n))
        for i in range(n):
            for j in range(i, n):
                K[i, j] = self.metric(self.X[i], self.X[j])
        K = np.triu(K) + np.triu(K, 1).T
        self.xd = np.diagonal(K).copy()
        if self.normalize:
            with np.errstate(invalid="ignore", divide="ignore"):
                return K / np.sqrt(np.outer(self.xd, self.xd))
        return K

    def transform(self, Y):
        Yp = self.parse(Y)
        K = np.array([[self.metric(y, x) for x in self.X] for y in Yp]).reshape(len(Yp), len(self.X))
        if self.normalize:
            yd = np.array([self.metric(y, y) for y in Yp])
            with np.errstate(invalid="ignore", divide="ignore"):
                K /= np.sqrt(np.outer(yd, self.xd))
        return K


# ---- numpy's summation order (umath loops: the pairwise sum of a contiguous float64 reduction)
def pairwise_sum(a):
    """numpy's pairwise_sum over a contiguous float64 block: below 8 elements a plain loop from -0.0, up to 128 eight
    accumulators combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)) then the tail, above that two halves
    split at a multiple of 8."""
    n = len(a)
    if n < 8:
        res = np.float64(-0.0)
        for x in a:
            res = res + x
        return res
    if n <= 128:
        r = [np.float64(x) for x in a[:8]]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                r[j] = r[j] + a[i + j]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for x in a[i:]:
            res = res + x
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def add_reduce(a):
    """np.sum of a 1-d float64 array (numpy 2): the pairwise sum of all its elements, added to the identity."""
    return pairwise_sum(np.asarray(a, dtype=np.float64))


def mean(a):
    """np.mean of a 1-d float64 array."""
    return add_reduce(a) / len(a)
