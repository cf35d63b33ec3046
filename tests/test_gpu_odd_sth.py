"""OddSth on the device: K equal with == to the real reference's goldens, the exported identity signatures rebuilding
the reference's feature keys and C, random sets against the CPU oracle, forced hash collisions through the retry,
counts >= 256 and K >= 2^24 exact, the routes (row ranges, device output) against each other, bit-identical repeats,
and the vertex cap at its edge."""
import json
import os
import sys

import numpy as np
import pytest

from grakel_b200 import Graph, GraphKernel, OddSth
from grakel_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import odd_oracle  # noqa: E402
from nspd_cases import _rand_graph  # noqa: E402
from odd_cases import GRAPH_OBJECT_CASES, cases, key_hash  # noqa: E402

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = np.load(os.path.join(HERE, "golden", "odd_sth.npz"))
CASES = {}
for _name, _X, _Y, _p in cases():
    if _name in GRAPH_OBJECT_CASES:
        _X = [Graph(x[0], x[1], {}) for x in _X]
        _Y = None if _Y is None else [Graph(y[0], y[1], {}) for y in _Y]
    CASES[_name] = (_X, _Y, _p)


def _eq(K, ref):
    return K.shape == ref.shape and np.array_equal(K, ref, equal_nan=True)


@pytest.mark.parametrize("name", json.loads(str(G["__cases__"])))
@pytest.mark.parametrize("norm", [0, 1])
def test_golden(name, norm):
    X, Y, p = CASES[name]
    k = OddSth(normalize=bool(norm), **p)
    K = k.fit_transform(X)
    if f"{name}/fit/{norm}" in G.files:
        ref = G[f"{name}/fit/{norm}"]
    else:  # the golden keeps only the unnormalised K: normalise it as odd_sth.py:169-171 does
        raw = G[f"{name}/fit/0"]
        d = np.diagonal(raw)
        ref = np.divide(raw, np.sqrt(np.outer(d, d)))
    assert _eq(K, ref), np.nanmax(np.abs(K - ref))
    assert k.stats_.gram_path == 14
    if Y is not None:
        Kt = k.transform(Y)
        assert _eq(Kt, G[f"{name}/transform/{norm}"]), np.nanmax(np.abs(Kt - G[f"{name}/transform/{norm}"]))
        xd, yd = k.diagonal()
        assert _eq(xd, G[f"{name}/xdiag/{norm}"]) and _eq(yd, G[f"{name}/ydiag/{norm}"])


def _identity_strings(est, label, off, child):
    """The reference's ID string of every exported identity, rebuilt from the signatures (children first)."""
    strs = est.X.dictionary
    out = [None] * len(label)

    def build(f):
        stack = [f]
        while stack:
            g = stack[-1]
            kids = child[off[g]:off[g + 1]]
            todo = [c for c in kids if out[c] is None]
            if todo:
                stack.extend(todo)
                continue
            stack.pop()
            s = strs[label[g]]
            out[g] = s + ("(" + ",".join(out[c] for c in kids) + ")" if len(kids) else "")
        return out[f]

    return [build(f) for f in range(len(label))]


@pytest.mark.parametrize("name", ["mutag_hNone", "mutag_h3", "directed_loops", "int_and_float", "strings", "isolated"])
def test_signatures_rebuild_reference_keys(name):
    X, _, p = CASES[name]
    k = OddSth(**p)
    k._keep_signatures = True
    k.fit_transform(X)
    label, off, child, C = k.signatures_
    keys = _identity_strings(k, label, off, child)
    assert len(set(keys)) == len(keys)
    assert {key_hash(s): int(c) for s, c in zip(keys, C)} == dict(zip(G[f"{name}/keys"].tolist(),
                                                                      G[f"{name}/C"].tolist()))
    assert k.stats_.n_columns == len(keys)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_sets_match_oracle(seed):
    rng = np.random.default_rng(100 + seed)
    X = [_rand_graph(rng, int(rng.integers(2, 16)), float(rng.uniform(0.1, 0.5)), 4, 1, directed=bool(seed % 2),
                     loops=seed == 2) for _ in range(30)]
    X = [[ed, nl] for ed, nl, _ in X]
    for h in (None, 1, 2, 4):
        k = OddSth(h=h)
        assert np.array_equal(k.fit_transform(X[:20]), odd_oracle.kernel(X[:20], None, h))
        assert np.array_equal(k.transform(X[20:]), odd_oracle.kernel(X[:20], X[20:], h))


def test_forced_collisions_take_the_retry():
    X, Y, p = CASES["mutag_h3"]
    ref = G["mutag_h3/fit/0"]
    k = OddSth(**p)
    with _lib.engine(None) as eng:
        eng.selftest_odd_collision(2)
    K = k.fit_transform(X)
    assert k.stats_.hash_retries == 2 and np.array_equal(K, ref)
    K = k.fit_transform(X)
    assert k.stats_.hash_retries == 0 and np.array_equal(K, ref)
    with _lib.engine(None) as eng:
        eng.selftest_odd_collision(1)
    assert np.array_equal(k.transform(Y), G["mutag_h3/transform/0"]) and k.stats_.hash_retries == 1


def _star(leaves, label=1):
    ed = {0: list(range(1, leaves + 1))}
    for i in range(1, leaves + 1):
        ed[i] = [0]
    return [ed, {i: label for i in range(leaves + 1)}]


def test_large_counts_exact():
    """Stars: the leaf identity '1' counts 2 * leaves per star (254, 256, 600), so the u8 panel, the bf16 panel and
    the CUDA-core route all run, and K reaches C phi^2 = 600^3 > 2^24."""
    X = [_star(127), _star(128), _star(300), _star(300), _star(5)]
    for h in (1, 2, None):
        k = OddSth(h=h)
        K = k.fit_transform(X)
        ref = odd_oracle.kernel(X, None, h)
        assert ref.max() > 2 ** 24 and np.array_equal(K, ref), h
        assert np.array_equal(k.transform(X[::-1]), odd_oracle.kernel(X, X[::-1], h))


def test_routes_agree(monkeypatch):
    X, Y, p = CASES["mutag_h2"]
    k = OddSth(**p)
    K = k.fit_transform(X)
    assert np.array_equal(K, G["mutag_h2/fit/0"])
    for _ in range(2):  # repeated runs are bit-identical
        assert np.array_equal(k.fit_transform(X), K)
    ids, rank = k.X.ids, k.X.rank
    Kr, _, _ = k._odd_run(k.X.block, ids, rank, len(X), row_range=(7, 31))
    assert np.array_equal(Kr, K[7:31])
    Kt = k.transform(Y)
    Kn = OddSth(normalize=True, **p)
    Kn.fit_transform(X)
    Ktn = Kn.transform(Y)
    assert np.array_equal(Ktn, G["mutag_h2/transform/1"])
    import torch
    dev = torch.zeros((len(X), len(X)), dtype=torch.float64, device="cuda")
    k._odd_run(k.X.block, ids, rank, len(X), device_ptr=dev.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), K)
    monkeypatch.setenv("GRAKEL_B200_ODD_C_BUDGET", str(8 * 40 * 8))  # a few rows per chunk
    assert np.array_equal(OddSth(**p).fit_transform(X), K)
    assert np.array_equal(OddSth(**p).fit(X).transform(Y), Kt)


def test_graph_kernel_dispatch():
    X, _, _ = CASES["random"]
    K = GraphKernel(kernel={"name": "ODD"}).fit_transform(X)
    assert np.array_equal(K, G["random/fit/0"])
    K = GraphKernel(kernel={"name": "odd_sth", "h": 2}, normalize=True).fit_transform(X)
    assert np.array_equal(K, G["random_h2/fit/1"])


def _path(n):
    ed = {i: [j for j in (i - 1, i + 1) if 0 <= j < n] for i in range(n)}
    return [ed, {i: i % 2 for i in range(n)}]


def test_vertex_cap_edge():
    X = [_path(4096), _path(6)]
    K = OddSth(h=2).fit_transform(X)
    assert np.array_equal(K, odd_oracle.kernel(X, None, 2))
    with pytest.raises(NotImplementedError):
        OddSth(h=2).fit_transform([_path(4097), _path(6)])
