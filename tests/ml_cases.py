"""MultiscaleLaplacian golden cases: the inputs are stored in tests/golden/multiscale_laplacian.npz beside the
reference's results, so the tests need nothing but that file."""
import os

import numpy as np


ERROR_CASES = [("gamma_negative", dict(gamma=-1.0)), ("heta_str", dict(heta="a")), ("L_negative", dict(L=-1)),
                ("L_float", dict(L=1.5)), ("P_zero", dict(P=0)), ("n_samples_zero", dict(n_samples=0)),
                ("int_labels", dict())]


def _sym(rs, n, p, weighted=False, loops=0):
    A = np.triu((rs.rand(n, n) < p).astype(float), 1)
    if weighted:
        A *= rs.randint(1, 4, size=(n, n))
    A = A + A.T
    for i in rs.choice(n, size=min(loops, n), replace=False):
        A[i, i] = float(rs.randint(1, 3))
    return A


def _rand_set(seed, n_graphs, lo, hi, dim, weighted=False, loops=0, integer=False, isolated=False):
    rs = np.random.RandomState(seed)
    out = []
    for g in range(n_graphs):
        n = int(rs.randint(lo, hi + 1))
        A = _sym(rs, n, 0.35, weighted, loops)
        if isolated and n > 2:
            A[n - 1, :] = A[:, n - 1] = 0.0
        phi = rs.randint(0, 5, size=(n, dim)).astype(np.int64) if integer else rs.rand(n, dim)
        out.append((A, phi))
    return out


def generated_cases(generate_dataset=None):
    """(name, X els, Y els, params, normalize variants); `generate_dataset` is the reference's generator (the golden
    script passes it), else that case is skipped."""
    cases = []
    if generate_dataset is not None:
        Xg, Yg = generate_dataset(n_graphs=100, r_vertices=(10, 20), r_connectivity=(0.4, 0.8), r_weight_edges=(1, 1),
                                  n_graphs_test=40, random_state=0, features=("na", 5))
        to_els = lambda G: [(np.asarray(g[0], dtype=float), np.array([list(g[1][i]) for i in range(len(g[1]))]))
                            for g in G]
        cases.append(("reference_tests", to_els(Xg), to_els(Yg), dict(random_state=0)))
    odd = _rand_set(3, 12, 1, 9, 4, weighted=True, loops=2, isolated=True)
    odd.append((np.zeros((1, 1)), np.array([[0.5, 0.25, 1.0, 2.0]])))
    cases += [
        ("weighted_loops", odd[:9], odd[9:], dict(random_state=1, L=2, P=3, n_samples=7)),
        ("integer_attrs", _rand_set(4, 10, 3, 8, 3, integer=True), _rand_set(5, 4, 3, 8, 3, integer=True),
         dict(random_state=2, L=1, P=10, n_samples=1000)),
        ("L0", _rand_set(6, 8, 2, 10, 6), _rand_set(7, 3, 2, 10, 6), dict(random_state=3, L=0, P=4)),
        ("L4_P1", _rand_set(8, 8, 3, 12, 5), _rand_set(9, 3, 3, 12, 5), dict(random_state=4, L=4, P=1, n_samples=1)),
        ("gamma_heta", _rand_set(10, 10, 4, 14, 5), _rand_set(11, 4, 4, 14, 5),
         dict(random_state=5, L=2, P=10, gamma=0.1, heta=0.5, n_samples=30)),
    ]
    return cases


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multiscale_laplacian.npz")


def _unpack(z, prefix):
    ns, A, phi = z[prefix + "_n"], z[prefix + "_A"], z[prefix + "_phi"]
    out, a, v = [], 0, 0
    for n in ns.tolist():
        out.append((A[a:a + n * n].reshape(n, n), phi[v:v + n]))
        a += n * n
        v += n
    return out


def load():
    """(meta, {case name: dict(X, Y, params, golden arrays by key)})."""
    import json
    z = np.load(GOLDEN)
    meta = json.loads(str(z["meta"]))
    cases = {}
    for c in meta["cases"]:
        name = c["name"]
        g = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "/")}
        cases[name] = dict(X=_unpack(z, name + "/X"), Y=_unpack(z, name + "/Y"), params=c["params"], gaps=c["gaps"],
                           levels=c["levels"], g=g)
    return meta, cases


def as_input(els):
    return [[A, {i: list(p[i]) for i in range(A.shape[0])}] for A, p in els]


def replay_eig(g, levels):
    """An eig that returns the reference's recorded (v, w) of the fit, call by call."""
    it = iter([(g["eig_v_%d" % l], g["eig_w_%d" % l]) for l in range(levels)])
    return lambda K: next(it)


def rel_err(K, R):
    return float(np.max(np.abs(K - R) / np.maximum(np.abs(R), 1e-300))) if R.size else 0.0
