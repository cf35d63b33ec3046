"""SvmTheta on the host: the oracle against the reference's goldens, the library's MT19937 draws against numpy, the
restated summation order, the schedule, validation errors and dispatch."""
import numpy as np
import pytest

import svmt_cases
import svmt_oracle as oracle
from grakel_b200 import GraphKernel, SvmTheta, _lib
from grakel_b200.kernels import svm_theta_inner, svmt_distribute

Z, INPUTS = svmt_cases.load()
SEEDED = [c for c in INPUTS if c + "/xg_m" in Z]


PARAMS = {c[0]: c[3] for c in svmt_cases.cases()}
PARAMS.update(reference_tests=dict(random_state=0), mutag=dict(random_state=1),
              mutag_6_8=dict(random_state=1, subsets_size_range=(6, 8)))


def _params(name):
    return PARAMS[name]


@pytest.mark.parametrize("name", SEEDED)
def test_oracle_matches_golden(name):
    X, Y = INPUTS[name]
    for key, G in (("xg", X), ("yg", Y)):
        m, alphas, iters = zip(*(oracle.theta_alphas(A) for A in G))
        assert np.array_equal(np.array(m), Z[f"{name}/{key}_m"])
        assert np.array_equal(np.concatenate(alphas), Z[f"{name}/{key}_alpha"])
        assert np.array_equal(np.array(iters), Z[f"{name}/{key}_iters"])
    for norm in (0, 1):
        o = oracle.SvmThetaOracle(normalize=bool(norm), **_params(name))
        assert np.array_equal(o.fit_transform(X), Z[f"{name}/fit/{norm}"], equal_nan=True)
        assert np.array_equal(o.transform(Y), Z[f"{name}/transform/{norm}"], equal_nan=True)


def test_draw_matches_numpy_choice():
    rs = np.random.RandomState(0)
    calls = [(int(n), int(k)) for n, k in zip(rs.randint(1, 129, 3000), rs.randint(1, 129, 3000)) if k <= n]
    ref = np.random.RandomState(123)
    mine = np.random.RandomState(123)
    for n, k in calls[:200]:  # one call per graph and level
        got = _lib.svmt_draw(mine, [n], k, [[1]])
        assert np.array_equal(got, ref.choice(n, k, replace=False))
    # many samples and levels at once, across MT19937 regenerations
    sizes = [n for n, _ in calls[200:600]]
    lo, L = 1, 128
    counts = rs.randint(0, 3, size=(len(sizes), L)).astype(np.int32)
    got = _lib.svmt_draw(mine, sizes, lo, counts)
    want = [ref.choice(n, lo + li, replace=False) for g, n in enumerate(sizes) for li in range(L)
            for _ in range(counts[g, li]) if lo + li <= n]
    assert np.array_equal(got, np.concatenate(want))
    a, b = mine.get_state(), ref.get_state()
    assert np.array_equal(a[1], b[1]) and a[2] == b[2] and a[3:] == b[3:]


def test_draw_keeps_gaussian_cache():
    rs = np.random.RandomState(5)
    rs.standard_normal()  # leaves a cached gaussian
    before = rs.get_state()
    _lib.svmt_draw(rs, [9], 3, [[4]])
    after = rs.get_state()
    assert after[3:] == before[3:] and after[3] == 1


@pytest.mark.parametrize("name", SEEDED)
def test_golden_draws_from_schedule(name):
    X, _ = INPUTS[name]
    p = _params(name)
    k = SvmTheta(**{q: v for q, v in p.items() if q != "random_state"})
    k.random_state = p["random_state"]
    k.initialize()
    sizes = np.array([A.shape[0] for A in X], dtype=np.int32)
    counts = k._schedule(sizes)
    idx = _lib.svmt_draw(k.random_state_, sizes, k.subsets_size_range[0], counts)
    assert np.array_equal(idx, Z[name + "/xg_drawn"])
    _, key, pos, _, _ = k.random_state_.get_state()
    assert np.array_equal(key, Z[name + "/state_fit_key"]) and pos == Z[name + "/state_fit_pos"]


def test_zero_division_after_earlier_draws():
    name, X, params = svmt_cases.ZERO_DIVISION
    k = SvmTheta(random_state=params["random_state"])
    k.initialize()
    with pytest.raises(ZeroDivisionError):
        k._schedule(np.array([A.shape[0] for A in X], dtype=np.int32))
    _, key, pos, _, _ = k.random_state_.get_state()
    assert np.array_equal(key, Z[name + "/state_key"]) and pos == Z[name + "/state_pos"]


@pytest.mark.parametrize("name", SEEDED)
def test_schedule_matches_reference(name):
    """The samples per subset size of every golden graph, as the reference's distribute_samples returned them."""
    p = _params(name)
    k = SvmTheta(**{q: v for q, v in p.items() if q != "random_state"})
    k.initialize()
    lo = k.subsets_size_range[0]
    for key, G in zip(("xg", "yg"), INPUTS[name]):
        sizes = np.array([A.shape[0] for A in G], dtype=np.int32)
        want = Z[f"{name}/{key}_sched"]
        assert np.array_equal(k._schedule(sizes), want)
        for n, row in zip(sizes, want):
            d = {lo + i: int(v) for i, v in enumerate(row) if v > 0}
            assert svmt_distribute(int(n), k.subsets_size_range, k.n_samples) == d
            assert oracle.distribute(int(n), k.subsets_size_range, k.n_samples) == d


def test_distribute_matches_oracle():
    for r in ((2, 8), (1, 3), (6, 8), (3, 14), (2, 70), (5, 5)):
        for n in range(1, 129):
            for ns in (1, 7, 50, 333, 1000):
                if n < r[0]:
                    with pytest.raises(ZeroDivisionError):
                        svmt_distribute(n, r, ns)
                else:
                    assert svmt_distribute(n, r, ns) == oracle.distribute(n, r, ns)


def test_summation_order_matches_numpy():
    rs = np.random.RandomState(7)
    for n in range(1, 301):
        for scale in (1.0, 1e-8, 1e8):
            a = rs.rand(n) * rs.choice([1.0, scale], n)
            assert oracle.add_reduce(a) == np.sum(a)
            assert oracle.mean(a) == np.mean(a)


@pytest.mark.parametrize("case", [c[0] for c in svmt_cases.ERROR_CASES])
def test_validation_errors(case):
    params = dict(svmt_cases.ERROR_CASES)[case]
    want = str(Z["error/" + case])
    with pytest.raises(Exception) as e:
        SvmTheta(**params).fit([[np.ones((3, 3))]])
    assert type(e.value).__name__ == want


def test_dispatch():
    for name in ("svm_theta", "SVMT"):
        gk = GraphKernel(kernel={"name": name, "n_samples": 7}, random_state=3)
        gk.initialize()
        assert type(gk.kernel_) is SvmTheta and gk.kernel_.n_samples == 7
        assert gk.kernel_.random_state is gk.random_state_
    gk = GraphKernel(kernel="SVMT")
    gk.initialize()
    assert gk.kernel_.random_state is None and gk.kernel_.metric is svm_theta_inner
    for name in ("lovasz_theta", "LOVT"):
        with pytest.raises(NotImplementedError):
            GraphKernel(kernel=name).initialize()
