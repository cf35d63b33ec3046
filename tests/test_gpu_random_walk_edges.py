"""RandomWalk / RandomWalkLabeled on the H100 at benchmark scale and at their numerical edges, against the NumPy / SciPy
restatement (tests/rw_oracle.py): every route on bench.gen_list(2000, 40, 0) with the CG iteration counts, the tuned
lamda, directed transforms, both sides of the shared-memory / global-workspace switch, the workspace's size, the
Taylor series on hub graphs (where M^k 1 overflows long before the series may stop) and the pair-index math of a
5 000-graph square."""
import contextlib
import os
import sys
import warnings

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import rw_oracle as O  # noqa: E402
from bench import gen_list  # noqa: E402
from grakel_b200 import RandomWalk, RandomWalkLabeled, _lib  # noqa: E402
from grakel_b200.packing import adjacency_and_labels  # noqa: E402

pytestmark = pytest.mark.gpu

CG_REL = 1e-12      # two summation orders of the same CG differ by ~1e-15 at these lamdas
TAYLOR_REL = 1e-11  # the documented Taylor bound
SMEM_MAX = 231424   # RW_SMEM_MAX: CG needs 24 n^2 bytes, the series 16 n^2


@pytest.fixture(scope="module")
def bench_graphs():
    """(the estimators' input, [(A, labels)] of RandomWalkLabeled, [(A, None)] of RandomWalk): the config-2 graphs."""
    X = gen_list(2000, 40, 0)
    return X, [adjacency_and_labels(g, L) for g, L in X], [(adjacency_and_labels(g)[0], None) for g, _ in X]


@pytest.fixture
def own_engine(monkeypatch):
    """A fresh engine for the estimators of the test, closed afterwards: its buffers start empty and are the only ones
    that grow while it runs."""
    eng = _lib.Engine()
    monkeypatch.setattr(_lib, "engine", lambda device=None: contextlib.nullcontext(eng))
    try:
        yield eng
    finally:
        eng.close()


def sample(n, n_off, seed, sizes=None):
    """Every diagonal entry, about n_off seeded off-diagonal entries and, with `sizes`, the ten largest graphs against
    each other."""
    rs = np.random.RandomState(seed)
    pairs = [(i, i) for i in range(n)]
    pairs += [(int(i), int(j)) for i, j in rs.randint(n, size=(n_off, 2)) if i != j]
    if sizes is not None:
        big = np.argsort(sizes, kind="stable")[-10:]
        pairs += [(int(i), int(j)) for i in big for j in big if i != j]
    return pairs


def check_cg(K, its, G, lam, pairs, labeled, transform=False):
    """K[i, j] against the oracle's CG on op(min, max) (transform: op(Y[i], X[j]), G = (Y, X)) and, where given, the
    device's iteration count against the oracle's.  A count may differ only where the oracle's ||r|| at the deciding
    norm test lies within 1e-9 relative of atol; K is then compared with the oracle run for the device's count."""
    for i, j in pairs:
        (A, La), (B, Lb) = (G[0][i], G[1][j]) if transform else (G[min(i, j)], G[max(i, j)])
        if not labeled:
            La = Lb = None
        v, it, norms, atol = O.cg_trace(A, B, lam, La, Lb)
        if its is not None and its[i, j] != it:
            k = min(int(its[i, j]), it)
            assert abs(its[i, j] - it) == 1 and abs(norms[k] - atol) <= 1e-9 * atol, (i, j, its[i, j], it)
            v = O.cg_trace(A, B, lam, La, Lb, iters=int(its[i, j]))[0]
        assert abs(K[i, j] - v) <= CG_REL * abs(v), (i, j, K[i, j], v)


# ---- benchmark scale -------------------------------------------------------------------------------------------------
def test_bench_cg(bench_graphs):
    """RandomWalk(lamda=0.01): the 2000 x 2000 Gram, its iteration counts, row ranges, device output and normalize."""
    torch = pytest.importorskip("torch")
    X, _, G = bench_graphs
    n = len(X)
    K = RandomWalk(lamda=0.01).fit_transform(X)
    eng = _lib.get_engine()
    its = eng.rw_iterations(n, n)
    assert np.array_equal(K, K.T) and np.all(np.isfinite(K))
    check_cg(K, its, G, 0.01, sample(n, 1000, 1, [A.shape[0] for A, _ in G]), False)
    for r0, r1 in ((1234, 1301), (n - 1, n)):  # a block from mid-matrix, and the last row
        Kb, _, _ = eng.gram(n, row_range=(r0, r1))
        assert np.array_equal(Kb, K[r0:r1]), (r0, r1)
    t = torch.full((n, n), float("nan"), dtype=torch.float64, device="cuda")
    eng.gram(n, device_ptr=t.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), K)
    del t
    Kn = RandomWalk(lamda=0.01, normalize=True).fit_transform(X)
    d = np.diag(K)
    assert np.allclose(Kn, K / np.sqrt(np.outer(d, d)), rtol=1e-14, atol=0)


def test_bench_cg_labeled(bench_graphs):
    X, G, _ = bench_graphs
    n = len(X)
    K = RandomWalkLabeled(lamda=0.01).fit_transform(X)
    its = _lib.get_engine().rw_iterations(n, n)
    assert np.array_equal(K, K.T) and np.all(np.isfinite(K))
    pairs = sample(n, 0, 2)[::20] + sample(n, 150, 2, [A.shape[0] for A, _ in G])[n:]
    check_cg(K, its, G, 0.01, pairs, True)


def test_bench_taylor_labeled(bench_graphs):
    X, G, _ = bench_graphs
    n = len(X)
    est = RandomWalkLabeled(lamda=0.01, kernel_type="exponential")
    K = est.fit_transform(X)
    assert est.stats_.rw_cap_hits == 0 and np.array_equal(K, K.T)
    for i, j in sample(n, 1000, 3, [A.shape[0] for A, _ in G]):
        (A, La), (B, Lb) = G[min(i, j)], G[max(i, j)]
        v = O.taylor_pair(A, B, 0.01, La, Lb)
        assert abs(K[i, j] - v) <= TAYLOR_REL * v, (i, j, K[i, j], v)
    # the oracle's series against dense expm on the smallest pairs
    small = np.argsort([A.shape[0] for A, _ in G], kind="stable")[:4]
    for i in small:
        for j in small:
            (A, La), (B, Lb) = G[i], G[j]
            ref = O.expm_pair(A, B, 0.01, La, Lb)
            assert abs(O.taylor_pair(A, B, 0.01, La, Lb) - ref) <= 1e-12 * ref
            assert abs(K[i, j] - ref) <= TAYLOR_REL * ref


def test_bench_spectral(bench_graphs):
    X, _, G = bench_graphs
    n = len(X)
    K = RandomWalk(lamda=0.01, kernel_type="exponential").fit_transform(X)
    qw = [O.eig_data(A) for A, _ in G]
    f = lambda z: np.exp(0.01 * z)
    for i, j in sample(n, 1000, 4, [A.shape[0] for A, _ in G]):
        s, mag = O.spectral_pair(*qw[min(i, j)], *qw[max(i, j)], f)
        assert abs(K[i, j] - s) <= 1e-12 * mag, (i, j, K[i, j], s)


# ---- the tuned lamda -------------------------------------------------------------------------------------------------
def test_tuned_lamda(bench_graphs):
    """lamda=1.0 diverges on the bench graphs: the fit lowers it to 0.9 / rho^2, the worst-conditioned solve allowed."""
    X, _, G = bench_graphs
    X, G = X[:300], G[:300]
    est = RandomWalk(lamda=1.0)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        K = est.fit_transform(X)
    radii = [float(np.max(np.absolute(np.linalg.eigvals(A)))) for A, _ in G]
    rho = max(radii)
    lam = 0.9 * (1.0 / rho ** 2)
    assert est._lamda == lam
    msgs = [str(x.message) for x in w if issubclass(x.category, RuntimeWarning)]
    assert msgs == ["lamda=1.0 makes the random walk series diverge on these graphs, whose largest spectral radius is "
                    "%s: convergence needs lamda < %s. Using lamda=%s instead. Pass a smaller lamda, or p=<int> for a "
                    "fixed number of steps, to silence this." % (format(rho, ".4g"), format(1 / rho ** 2, ".4g"),
                                                                  format(lam, ".4g"))]
    its = _lib.get_engine().rw_iterations(300, 300)
    assert np.array_equal(K, K.T) and np.all(np.isfinite(K))
    check_cg(K, its, G, lam, sample(300, 300, 5, radii), False)
    assert its.max() >= 10  # the solves are harder than at the default lamda


# ---- directed graphs, fit and transform orientation ------------------------------------------------------------------
def test_directed_transform_orientation(bench_graphs):
    """Fit entries are op(min, max), transform entry (j, i) is op(Y[j], X[i]); on directed graphs the CG of the swapped
    pair differs from it well beyond the bound, so the order is pinned."""
    _, _, G = bench_graphs
    rs = np.random.RandomState(9)
    D = []
    for A, _ in G:
        U = np.triu(A, 1)
        flip = np.triu(rs.rand(*A.shape) < 0.5, 1) & (U != 0)
        D.append((np.where(flip, 0.0, U) + np.where(flip, U, 0.0).T, None))
    Xd, Yd = D[:1500], D[1500:]
    est = RandomWalk(lamda=0.01)
    K = est.fit_transform([[A] for A, _ in Xd])
    assert est._lamda == 0.01
    check_cg(K, None, Xd, 0.01, sample(1500, 200, 6)[::15], False)
    Kt = est.transform([[A] for A, _ in Yd])
    assert Kt.shape == (500, 1500)
    rs = np.random.RandomState(7)
    pairs = [(int(j), int(i)) for j, i in zip(rs.randint(500, size=300), rs.randint(1500, size=300))]
    check_cg(Kt, None, (Yd, Xd), 0.01, pairs, False, transform=True)
    swapped = [abs(O.cg_pair(Xd[i][0], Yd[j][0], 0.01)[0] - Kt[j, i]) > 1e3 * CG_REL * abs(Kt[j, i])
               for j, i in pairs[:40]]
    assert sum(swapped) >= 10


# ---- shared memory and the global workspace --------------------------------------------------------------------------
def _graph(n, seed, n_labels=3):
    rs = np.random.RandomState(seed)
    A = np.triu((rs.rand(n, n) < 4.0 / (n - 1)).astype(float), 1)
    return A + A.T, [int(x) for x in rs.randint(n_labels, size=n)]


def _as_input(G, labeled):
    return [[A, dict(enumerate(L))] if labeled else [A] for A, L in G]


def _oracle(est, A, La, B, Lb):
    """(value, bound) of one pair on the estimator's route."""
    lab = isinstance(est, RandomWalkLabeled)
    La, Lb = (La, Lb) if lab else (None, None)
    route, fn = est._route()
    if route == _lib.GK_RW_CG:
        v = O.cg_pair(A, B, est._lamda, La, Lb)[0]
        return v, CG_REL * abs(v)
    if fn == _lib.GK_RW_EXP:
        v = O.taylor_pair(A, B, est._lamda, La, Lb)
        return v, TAYLOR_REL * abs(v)
    v, mag = O.series_pair(A, B, est.mu_, La, Lb)
    return v, 1e-12 * mag


def _live():
    return _lib.live_bytes()[0]


SWITCH = [("cg", RandomWalk, dict(lamda=0.01), 3, 98),
          ("cg_labeled", RandomWalkLabeled, dict(lamda=0.01), 3, 98),
          ("taylor_labeled", RandomWalkLabeled, dict(lamda=0.01, kernel_type="exponential"), 2, 120),
          ("finite_series", RandomWalk, dict(lamda=0.01, p=3, method_type="baseline"), 2, 120)]


@pytest.mark.parametrize("name,cls,params,nvec,n", SWITCH, ids=[s[0] for s in SWITCH])
def test_shared_memory_and_workspace_agree(own_engine, name, cls, params, nvec, n):
    """The largest graph of a square launch at the last size whose vectors fit in shared memory, then one vertex more:
    the launch spills to the workspace (which grows by a slice per pair) and the smaller pairs keep their bits."""
    assert 8 * nvec * n * n <= SMEM_MAX < 8 * nvec * (n + 1) ** 2
    lab = cls is RandomWalkLabeled
    G = [_graph(n, 1), _graph(60, 2), _graph(30, 3), _graph(n + 1, 4)]
    est = cls(**params)
    K1 = est.fit_transform(_as_input(G[:3], lab))
    b1 = _live()
    K2 = cls(**params).fit_transform(_as_input(G, lab))
    b2 = _live()
    assert np.array_equal(K2[:3, :3], K1)
    # 10 pairs of the square, each on a workspace slice of its own; had the first launch spilled too, its 6 slices
    # would already be held
    assert b2 - b1 >= 10 * 8 * nvec * (n + 1) ** 2, (b1, b2)
    for i in range(4):
        for j in range(i, 4):
            (A, La), (B, Lb) = G[i], G[j]
            v, tol = _oracle(est, A, La, B, Lb)
            assert abs(K2[i, j] - v) <= tol, (i, j, K2[i, j], v)


def test_transform_launch_switch(own_engine):
    """A transform launch is sized by its rows times its columns: 98-vertex fit graphs with a 98-vertex transform graph
    fit in shared memory, a 99-vertex transform graph spills."""
    X = [_graph(98, 11), _graph(60, 12)]
    Y = [_graph(98, 13), _graph(30, 14)]
    big = _graph(99, 15)
    for cls in (RandomWalk, RandomWalkLabeled):
        lab = cls is RandomWalkLabeled
        est = cls(lamda=0.01)
        est.fit(_as_input(X, lab))
        Kt1 = est.transform(_as_input(Y, lab))
        b1 = _live()
        Kt2 = est.transform(_as_input(Y + [big], lab))
        b2 = _live()
        assert np.array_equal(Kt2[:2], Kt1)
        if not lab:  # the workspace only grows: the second class reuses it
            assert b2 - b1 >= 6 * 24 * 99 * 98, (b1, b2)
        check_cg(Kt2, None, (Y + [big], X), 0.01, [(j, i) for j in range(3) for i in range(2)], lab, transform=True)


def test_workspace_is_bounded(own_engine, bench_graphs):
    """A 600-vertex graph needs an 8.6 MB CG slice: alone it holds one slice per launch, not one per possible CTA, and
    among 50 bench graphs the workspace stays within 1 GiB."""
    _, _, G = bench_graphs
    A = np.triu((np.random.RandomState(21).rand(600, 600) < 4.0 / 599).astype(float), 1)
    A = A + A.T
    b0 = _live()
    K = RandomWalk(lamda=0.01).fit_transform([[A]])
    alone = _live() - b0
    assert alone <= 20 << 20, alone
    v, _ = O.cg_pair(A, A, 0.01)
    assert abs(K[0, 0] - v) <= CG_REL * v
    H = G[:50] + [(A, None)]
    b0 = _live()
    K = RandomWalk(lamda=0.01).fit_transform([[B] for B, _ in H])
    among = _live() - b0
    assert among <= (1 << 30) + (64 << 20), among
    its = own_engine.rw_iterations(51, 51)
    check_cg(K, its, H, 0.01, [(i, 50) for i in range(51)] + [(i, i) for i in range(50)], False)


# ---- the Taylor series on hub graphs ---------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hub_reference():
    """[(A, 1^T expm(0.1 kron(A_i, A_j)) 1)]: dense expm up to 3 600 rows, the eigh form beyond."""
    G = list(O.hub_graphs().values())
    ref = np.zeros((len(G), len(G)))
    for i, A in enumerate(G):
        for j, B in enumerate(G):
            if j >= i:
                big = A.shape[0] * B.shape[0] > 3600
                ref[i, j] = ref[j, i] = O.symmetric_expm_pair(A, B, 0.1) if big else O.expm_pair(A, B, 0.1)
    return G, ref


@pytest.mark.parametrize("labeled", [True, False], ids=["labeled_fast", "baseline"])
def test_taylor_hub_graphs(hub_reference, labeled):
    """K31, a vertex of degree 40 in 60 and a 100-leaf star: M^k 1 reaches inf before k >= 2 lamda R_i R_j while
    lamda^k / k! underflows.  The series carries the scaled vector, so K is finite, within the Taylor bound and never at
    the term cap."""
    G, ref = hub_reference
    if labeled:
        make = lambda **kw: RandomWalkLabeled(lamda=0.1, kernel_type="exponential", **kw)
        X = [[A, {v: 0 for v in range(A.shape[0])}] for A in G]
    else:
        make = lambda **kw: RandomWalk(lamda=0.1, method_type="baseline", kernel_type="exponential", **kw)
        X = [[A] for A in G]
    est = make()
    K = est.fit_transform(X)
    assert est.stats_.rw_cap_hits == 0
    assert np.all(np.isfinite(K)) and np.all(np.abs(K - ref) <= TAYLOR_REL * ref), np.abs(K - ref) / ref
    Kn = make(normalize=True).fit_transform(X)
    assert np.all(np.isfinite(Kn))
    assert np.allclose(Kn, K / np.sqrt(np.outer(np.diag(K), np.diag(K))), rtol=1e-14, atol=0)


# ---- the pair index at large N ---------------------------------------------------------------------------------------
def _shapes():
    one = np.zeros((1, 1))
    edge = np.array([[0.0, 1.0], [1.0, 0.0]])
    path = np.zeros((3, 3))
    path[0, 1] = path[1, 2] = 1.0  # directed 0 -> 1 -> 2
    tri = np.ones((3, 3)) - np.eye(3)
    star = np.zeros((4, 4))
    star[0, 1:] = star[1:, 0] = 1.0
    return [one, edge, path, tri, star, np.zeros((2, 2))]


def test_pair_index_at_large_n():
    """5 000 graphs of six tiny shapes: each of the 12.5 M entries of the mirrored upper triangle, and of a row block,
    is the device's value of op(shape of min(i, j), shape of max(i, j)), bit for bit."""
    S = _shapes()
    est = RandomWalk(lamda=0.1)
    est.fit([[A] for A in S])
    T = est.transform([[A] for A in S])  # T[a, b] = op(S[a], S[b]), both orders
    for a in range(6):
        for b in range(6):
            v, _ = O.cg_pair(S[a], S[b], 0.1)
            assert abs(T[a, b] - v) <= CG_REL * abs(v), (a, b)
    n = 5000
    s = np.random.RandomState(3).randint(6, size=n)
    K = RandomWalk(lamda=0.1).fit_transform([[S[k]] for k in s])
    assert K.shape == (n, n)
    lo = T[s[:, None], s[None, :]]  # op(X[i], X[j]) for every i, j
    for r0 in range(0, n, 500):
        r1 = min(n, r0 + 500)
        i, j = np.arange(r0, r1)[:, None], np.arange(n)[None, :]
        want = np.where(i <= j, lo[r0:r1], lo[:, r0:r1].T)
        assert np.array_equal(K[r0:r1], want), r0
    Kb, _, _ = _lib.get_engine().gram(n, row_range=(2345, 2467))
    assert np.array_equal(Kb, K[2345:2467])
