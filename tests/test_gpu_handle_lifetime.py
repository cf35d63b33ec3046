"""Lifetime of the engine handle: destroying a handle frees every buffer it allocated, engines created and used from
several threads at once compute what they compute one after the other, and the Gram self-test frees its scratch.

The estimators run here on engines the test creates and closes (`_lib.engine` is pointed at them): the pool behind
`_lib.engine` never closes its engines, and a fresh engine is what a handle's first use, the state under test, needs.
Every feature family's C-ABI sequence (pack -> *_features -> gram, square by fit_transform and with n_fit < N by
transform) then runs through the Engine's methods on inputs the estimators build."""
import contextlib
import os
import sys
import threading

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

from bench import gen_list  # noqa: E402
from ml_cases import _rand_set  # noqa: E402
from nspd_cases import mutag  # noqa: E402
from oracle.gk_oracle import gen  # noqa: E402
from grakel_b200 import (CoreFramework, EdgeHistogram, GraphHopper, GraphletSampling, HadamardCode,  # noqa: E402
                         MultiscaleLaplacian, NeighborhoodHash, NeighborhoodSubgraphPairwiseDistance, OddSth,
                         Propagation, PropagationAttr, PyramidMatch, RandomWalk, RandomWalkLabeled, ShortestPath,
                         ShortestPathAttr, SubgraphMatching, SvmTheta, VertexHistogram, WeisfeilerLehman,
                         WeisfeilerLehmanOptimalAssignment, _lib)

pytestmark = pytest.mark.gpu

_local = threading.local()


@pytest.fixture
def own_engines(monkeypatch):
    """Estimator runs on the calling thread use `_local.eng` instead of an engine of the pool."""
    monkeypatch.setattr(_lib, "engine", lambda device=None: contextlib.nullcontext(_local.eng))


def _run(est, X, Y):
    """fit_transform(X), then transform(Y) when given: the square and the n_fit < N Gram of one family."""
    K = est.fit_transform(X)
    return K if Y is None else (K, est.transform(Y))


def _split(X, n_fit):
    return X[:n_fit], X[n_fit:]


def _families():
    lab = _split(gen(30, 10, 1), 22)
    adj = _split(gen(30, 10, 2, as_adj=True), 22)
    attr = _split(gen(24, 9, 3, attr=3, as_adj=True), 18)
    mut = _split(mutag()[:30], 22)
    ml = (_rand_set(1, 10, 3, 8, 3), _rand_set(2, 4, 3, 8, 3))
    return [
        ("wl", lambda: WeisfeilerLehman(n_iter=3), lab),
        ("vh", lambda: VertexHistogram(), lab),
        ("eh", lambda: EdgeHistogram(), mut),
        ("wl_eh", lambda: WeisfeilerLehman(n_iter=2, base_graph_kernel=EdgeHistogram), mut),
        ("wl_oa", lambda: WeisfeilerLehmanOptimalAssignment(n_iter=3), lab),
        ("sp", lambda: ShortestPath(), adj),
        ("wl_sp", lambda: WeisfeilerLehman(n_iter=2, base_graph_kernel=ShortestPath), adj),
        ("spattr", lambda: ShortestPathAttr(), attr),
        ("gh_linear", lambda: GraphHopper(kernel_type="linear"), attr),
        ("gh_gaussian", lambda: GraphHopper(kernel_type=("gaussian", 0.5)), attr),
        ("nh", lambda: NeighborhoodHash(R=3, random_state=0), lab),
        ("rw", lambda: RandomWalk(lamda=0.01), adj),
        ("rw_labeled", lambda: RandomWalkLabeled(lamda=0.01), adj),
        ("pk", lambda: Propagation(random_state=0), lab),
        ("pk_attr", lambda: PropagationAttr(random_state=0), attr),
        ("pm", lambda: PyramidMatch(with_labels=True), lab),
        ("wl_pm", lambda: WeisfeilerLehman(n_iter=2, base_graph_kernel=(PyramidMatch, {"with_labels": True})), lab),
        ("hc", lambda: HadamardCode(n_iter=3), lab),
        ("nspd", lambda: NeighborhoodSubgraphPairwiseDistance(), mut),
        ("wl_nspd", lambda: WeisfeilerLehman(n_iter=2, base_graph_kernel=NeighborhoodSubgraphPairwiseDistance), mut),
        ("sm", lambda: SubgraphMatching(k=3), mut),
        ("wl_sm", lambda: WeisfeilerLehman(n_iter=2, base_graph_kernel=(SubgraphMatching, {"k": 3})), mut),
        ("odd", lambda: OddSth(), mut),
        ("wl_odd", lambda: WeisfeilerLehman(n_iter=2, base_graph_kernel=OddSth), mut),
        ("ml", lambda: MultiscaleLaplacian(random_state=0), ml),
        ("svmt", lambda: SvmTheta(random_state=0), lab),
        ("gs", lambda: GraphletSampling(k=4, sampling={"n_samples": 40}, random_state=0), lab),
        ("core_sp", lambda: CoreFramework(base_graph_kernel=ShortestPath), adj),
    ]


def test_destroy_frees_every_buffer(own_engines):
    families = _families()
    before = _lib.live_bytes()
    _local.eng = _lib.Engine()
    try:
        for _, make, (X, Y) in families:
            _run(make(), X, Y)
        assert _lib.live_bytes()[0] > before[0]  # the engine's buffers are counted while it lives
    finally:
        _local.eng.close()
    assert _lib.live_bytes() == before


# one family per thread, each on a handle of its own: the C-ABI state of a handle's first use is set up concurrently
_CONCURRENT = [
    ("wl", lambda: WeisfeilerLehman(n_iter=3), gen_list(300, 12, 1)),
    ("sp", lambda: ShortestPath(), gen_list(300, 12, 2, as_adj=True)),
    ("nh", lambda: NeighborhoodHash(R=3, random_state=0), gen_list(300, 12, 3)),
    ("sm", lambda: SubgraphMatching(k=3, ke=None), [[g, L, dict.fromkeys(g, 0)] for g, L in gen_list(200, 12, 4)]),
]


def _fresh_run(make, X):
    _local.eng = _lib.Engine()
    try:
        return _run(make(), X[:-40], X[-40:])
    finally:
        _local.eng.close()


def test_concurrent_engines_match_serial(own_engines):
    serial = [_fresh_run(make, X) for _, make, X in _CONCURRENT]
    out, errors = [None] * len(_CONCURRENT), []
    start = threading.Barrier(len(_CONCURRENT))

    def worker(i):
        try:
            make, X = _CONCURRENT[i][1:]
            start.wait()
            out[i] = _fresh_run(make, X)
        except BaseException as e:  # surfaced below, on the test's thread
            errors.append((_CONCURRENT[i][0], e))

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(_CONCURRENT))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for (name, _, _), (K, Kt), (Ks, Kts) in zip(_CONCURRENT, out, serial):
        assert np.array_equal(K, Ks) and np.array_equal(Kt, Kts), name


def test_selftest_gram_frees_its_scratch():
    eng = _lib.Engine()
    try:
        counts = np.random.default_rng(5).integers(0, 4, size=(96, 200)).astype(np.uint16)
        before = _lib.live_bytes()
        a, b = eng.selftest_gram(counts)
        assert _lib.live_bytes() == before
        ref = counts.astype(np.float64) @ counts.T.astype(np.float64)
        assert np.array_equal(a, ref) and np.array_equal(b, ref)
    finally:
        eng.close()
