"""NeighborhoodSubgraphPairwiseDistance, OddSth and SubgraphMatching on the device at the benchmark's graph sizes
(bench.gen_list(·, 40, 0): 20-60 vertices) and past the sizes their goldens reach, bit for bit against the in-repo
restatements (nspd_oracle, odd_oracle, sm_oracle).  The restatements are cached per module; they take most of the
file's time."""
import os
import sys

import numpy as np
import pytest

from grakel_b200 import NeighborhoodSubgraphPairwiseDistance, OddSth, SubgraphMatching
from grakel_b200 import _lib
from grakel_b200.kernels import _nspd_graph

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "tools"))
import nspd_oracle  # noqa: E402
import odd_oracle  # noqa: E402
import sm_oracle  # noqa: E402
from bench_nspd import gen_workload  # noqa: E402

pytestmark = pytest.mark.gpu


def _directed(X, seed, loop_p):
    """One direction of every undirected edge, kept at random, and a self-loop on a share of the vertices."""
    rng = np.random.default_rng(seed)
    out = []
    for x in X:
        g, L = x[0], x[1]
        e = {}
        for (u, v) in sorted(g):
            if u < v:
                a, b = (u, v) if rng.random() < 0.5 else (v, u)
                e[(a, b)] = 1
        for v in L:
            if rng.random() < loop_p:
                e[(v, v)] = 1
        out.append([e, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in e}] if len(x) == 3 else [e, L])
    return out


def _hashes(graphs, r, d):
    """gk_nspd_hashes of every rho for the parsed graphs, [r + 1, V]."""
    k = NeighborhoodSubgraphPairwiseDistance(r=r, d=d)
    gp, rp, ci, lab, el, sh, tokens = k._pack(graphs)
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, lab, None, None)
        eng.nspd_features(r, d, sh, el, tokens)
        return np.stack([eng.nspd_hashes(rho, len(lab)) for rho in range(r + 1)])


# ---- NeighborhoodSubgraphPairwiseDistance: the benchmark workload (r = 3, d = 4)
@pytest.fixture(scope="module")
def nspd_bench():
    W = gen_workload(40)
    X, Y = W[:32], W[32:]
    ref = {}
    for norm in (0, 1):
        ref["fit", norm] = nspd_oracle.fit_transform(X, 3, 4, bool(norm))
        ref["transform", norm] = nspd_oracle.transform(X, Y, 3, 4, bool(norm))
    return X, Y, ref, nspd_oracle.vertex_hashes(X, 3, 4)


@pytest.mark.parametrize("norm", [0, 1])
def test_nspd_bench_workload(nspd_bench, norm):
    X, Y, ref, _ = nspd_bench
    k = NeighborhoodSubgraphPairwiseDistance(normalize=bool(norm))
    assert np.array_equal(k.fit_transform(X), ref["fit", norm])
    assert np.array_equal(k.transform(Y), ref["transform", norm])


def test_nspd_bench_hashes_and_routes(nspd_bench):
    X, _, ref, H = nspd_bench
    k = NeighborhoodSubgraphPairwiseDistance().fit(X)
    assert np.array_equal(_hashes(k.X, 3, 4), H)
    K = ref["fit", 0]
    Ks, _, _ = k._nspd_run(k.X, len(X), simt=True)
    assert np.array_equal(Ks, K)
    Kr, _, _ = k._nspd_run(k.X, len(X), row_range=(5, 27))
    assert np.array_equal(Kr, K[5:27])
    import torch
    dev = torch.zeros((len(X), len(X)), dtype=torch.float64, device="cuda")
    k._nspd_run(k.X, len(X), device_ptr=dev.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(dev.cpu().numpy(), K)


def test_nspd_directed_with_loops():
    """One direction of each edge and self-loops (the root listed twice in its radius-1 ball), r = 2, d = 3."""
    W = _directed(gen_workload(24), 7, 0.15)
    X, Y = W[:18], W[18:]
    k = NeighborhoodSubgraphPairwiseDistance(r=2, d=3)
    assert np.array_equal(k.fit_transform(X), nspd_oracle.fit_transform(X, 2, 3))
    assert np.array_equal(k.transform(Y), nspd_oracle.transform(X, Y, 2, 3))
    assert np.array_equal(_hashes(k.X, 2, 3), nspd_oracle.vertex_hashes(X, 2, 3))


def test_nspd_labels_sorting_as_strings():
    """Tokens str(delta) + "," + str(label) rank in string order: "1,10" < "1,2", "0,-1" < "0,0", and multi-digit
    edge labels; vertex labels that only the transformed graphs carry get ranks too."""
    from bench import gen_list
    rng = np.random.default_rng(11)
    pool = [-3, -1, 0, 1, 2, 9, 10, 11, 12, 100]
    W = []
    for g, L in gen_list(12, 40, 3):
        L = {v: int(rng.choice(pool[:-1])) for v in L}
        W.append([g, L, {e: int(rng.integers(12)) for e in g}])
    for g, L, _ in W[9:]:
        L[0] = 100
    X, Y = W[:9], W[9:]
    k = NeighborhoodSubgraphPairwiseDistance()
    assert np.array_equal(k.fit_transform(X), nspd_oracle.fit_transform(X))
    assert np.array_equal(k.transform(Y), nspd_oracle.transform(X, Y))
    assert np.array_equal(_hashes(k.X, 3, 4), nspd_oracle.vertex_hashes(X))


# ---- NSPD sets past the x2 growth branch: r = 2, d = 0 on near-complete digraphs
def _dense_graph(n, missing, loops, seed):
    """A complete digraph on n vertices without the out-edges `missing` {v: [w, ...]}, with self-loops on `loops`."""
    rng = np.random.default_rng(seed)
    L = {v: int(rng.integers(5)) for v in range(n)}
    gone = {(v, w) for v, ws in missing.items() for w in ws}
    e = {(u, v): 1 for u in range(n) for v in range(n) if (u != v or u in loops) and (u, v) not in gone}
    return [e, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in e}]


def _restated_hashes(graph, N, dp, v):
    """H[rho, v] for rho = 2, 1, 0 as nspd_oracle.hashes computes them (each sub-edge set a set comprehension over
    the previous one), with set membership for the ball."""
    n, edges, vl, el = graph
    elab = dict(zip(edges, el))
    re, out = sorted(edges), {}
    for rho in (2, 1, 0):
        sub = sorted(N[rho][v])
        inside = set(sub)
        re = {(i, j) for (i, j) in re if i in inside and j in inside}
        lab = {}
        parts = []
        for i in sub:
            s = "|".join(sorted(str(dp[(i, j)]) + "," + vl[j] for j in sub if (i, j) in dp))
            parts.append(s + ".")
            lab[i] = s
        enc = "".join(parts)[:-1] + ":" + "".join(lab[i] + "," + lab[j] + "," + elab[(i, j)] + "_" for (i, j) in re)
        out[rho] = nspd_oracle.aphash(enc)
    return out


def _root_hashes(graph):
    """H[0, v] of every vertex: the ball is {v}, its sub-edge set the self-loop when v has one."""
    n, edges, vl, el = graph
    loop = {i: el[k] for k, (i, j) in enumerate(edges) if i == j}
    out = []
    for v in range(n):
        s = "0," + vl[v]
        out.append(nspd_oracle.aphash(s + ":" + (s + "," + s + "," + loop[v] + "_" if v in loop else "")))
    return out


@pytest.fixture(scope="module")
def nspd_big():
    """Graphs of 398 vertices (157 924 directed edges, past inserts 78 643 and 157 286) and 281 vertices (78 680, past
    78 643) among small ones.  At rho = 2 the ball is the whole graph; at rho = 1 it is a vertex and its out-
    neighbours, so vertices 3 and 5 (out-edges removed) and 7 (a self-loop) differ from the others."""
    small = gen_workload(3)
    big = _dense_graph(398, {3: [0, 1, 2, 10], 5: list(range(100, 180))}, {7, 11}, 1)
    mid = _dense_graph(281, {}, {2}, 2)
    X = [small[0], big, small[1], mid, small[2]]
    parsed = [_nspd_graph(*x) for x in X]
    chosen = {1: [0, 3, 5, 7, 397], 3: [0, 2, 280]}
    ref = []
    for gi, graph in enumerate(parsed):
        if gi in chosen:
            N, _, dp = nspd_oracle.neighborhoods(graph[0], graph[1], 2, 0)
            ref.append({v: _restated_hashes(graph, N, dp, v) for v in chosen[gi]})
            ref[-1]["H0"] = _root_hashes(graph)
        else:
            ref.append(nspd_oracle.vertex_hashes([X[gi]], 2, 0))
    return X, parsed, ref


@pytest.mark.parametrize("slots", [None, 16])
def test_nspd_sets_past_doubling(nspd_big, slots, monkeypatch):
    """All five graphs at the default workspace budget; the 281-vertex graph among the small ones with the budget
    cut to 16 slots (GRAKEL_B200_NSPD_WS_BUDGET), so that each slot hashes vertices of graphs of every size in turn."""
    X, parsed, ref = nspd_big
    pick = [0, 1, 2, 3, 4] if slots is None else [0, 2, 3, 4]
    parsed, ref = [parsed[i] for i in pick], [ref[i] for i in pick]
    if slots:  # nspd_slot_words of the largest graph
        max_n = max(g[0] for g in parsed)
        max_e = max(len(g[1]) for g in parsed)
        cap = 16
        while cap <= 4 * max_e:
            cap *= 2
        words = 2 * cap + 2 * max_e + 3 * (max_n + 2) + max_n + (max_n + 1) ** 2
        monkeypatch.setenv("GRAKEL_B200_NSPD_WS_BUDGET", str(slots * words * 4))
    H = _hashes(parsed, 2, 0)
    v0 = 0
    for graph, want in zip(parsed, ref):
        n = graph[0]
        got = H[:, v0:v0 + n]
        if isinstance(want, dict):
            assert np.array_equal(got[0], np.array(want["H0"], dtype=np.uint32))
            for v, hv in want.items():
                if v != "H0":
                    assert [int(got[rho, v]) for rho in (2, 1, 0)] == [hv[2], hv[1], hv[0]], (n, v)
            # every vertex without a loop or a removed out-edge has the whole graph as its radius-1 ball, as vertex 0
            outdeg = np.bincount([i for i, j in graph[1] if i != j], minlength=n)
            loops = {i for i, j in graph[1] if i == j}
            plain = [v for v in range(n) if outdeg[v] == n - 1 and v not in loops]
            assert len(plain) > n - 5 and (got[1, plain] == want[0][1]).all() and (got[2] == want[0][2]).all()
        else:
            assert np.array_equal(got, want)
        v0 += n


def test_nspd_refuses_65535_vertices_before_allocating():
    """r > 0 with a graph of 65 535 vertices: the u32 label offsets of its ball cannot hold B^2.  The estimator
    refuses before packing, and the device library before it sizes the 5 n^2 bytes (21 GB) of level matrices."""
    import torch
    n = 65535
    g = (n, [], ["0"] * n, [])
    k = NeighborhoodSubgraphPairwiseDistance(r=1, d=0)
    with pytest.raises(NotImplementedError, match="65535"):
        k._nspd_run([g], 1)
    gp, rp, ci, lab, el, sh, tokens = k._pack([g])
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, lab, None, None)
        free0 = torch.cuda.mem_get_info()[0]
        with pytest.raises(NotImplementedError, match="65535"):
            eng.nspd_features(1, 0, sh, el, tokens)
        # the engine keeps what it sized until it closes: nothing near the 4 GiB level matrix was taken
        assert free0 - torch.cuda.mem_get_info()[0] < (2 << 30)


# ---- OddSth: the benchmark workload and the warps-per-CTA steps
@pytest.fixture(scope="module")
def odd_bench():
    from bench import gen_list
    X = gen_list(2000, 40, 0)
    return X, {h: odd_oracle.features(X, h) for h in (None, 2)}


@pytest.mark.parametrize("h", [None, 2])
def test_odd_bench_workload(odd_bench, h):
    X, phis = odd_bench
    px = phis[h]
    k = OddSth(h=h)
    assert np.array_equal(k.fit_transform(X), odd_oracle.gram(px))
    assert k.stats_.hash_retries == 0
    k = OddSth(h=h).fit(X[:1500])
    assert np.array_equal(k.transform(X[1500:]), odd_oracle.gram(px[:1500], px[1500:]))
    assert k.stats_.hash_retries == 0
    kn = OddSth(h=h, normalize=True)
    assert np.array_equal(kn.fit_transform(X), odd_oracle.gram(px, normalize=True))
    assert np.array_equal(kn.transform(X[:300]), odd_oracle.gram(px, px[:300], normalize=True))


def _tree(n, seed):
    """A random tree on n vertices (each vertex hangs off one of the 8 before it), labels 0-2."""
    rng = np.random.default_rng(seed)
    ed = {i: [] for i in range(n)}
    for v in range(1, n):
        u = int(rng.integers(max(0, v - 8), v))
        ed[u].append(v)
        ed[v].append(u)
    return [ed, {i: int(rng.integers(3)) for i in range(n)}]


@pytest.mark.parametrize("n, warps", [(342, 4), (1420, 4), (1421, 3), (1896, 3), (1897, 2)])
def test_odd_warp_steps(odd_bench, n, warps):
    """One tree added to the bench graphs sets the warps per CTA, min(4, 200 KiB / (n_pad * 36)), for every graph;
    from 342 vertices the launch needs the opt-in shared memory."""
    n_pad = (n + 3) // 4 * 4
    assert min(4, (200 << 10) // (n_pad * 36)) == warps
    X, phis = odd_bench
    T = _tree(n, n)
    Xs = X[:1000] + [T] + X[1000:]
    px = phis[None][:1000] + odd_oracle.features([T], None) + phis[None][1000:]
    assert np.array_equal(OddSth().fit_transform(Xs), odd_oracle.gram(px))


def test_odd_directed_with_loops(odd_bench):
    X = _directed(odd_bench[0][:300], 5, 0.1)
    px = odd_oracle.features(X, None)
    k = OddSth()
    assert np.array_equal(k.fit_transform(X[:240]), odd_oracle.gram(px[:240]))
    assert np.array_equal(k.transform(X[240:]), odd_oracle.gram(px[:240], px[240:]))


# ---- SubgraphMatching: bench graphs with edge labels (records in global memory), without (staged), directed
def _counts(k, graphs, n_fit, row):
    gp, rp, ci, ids, elids, vt, et, flags = k._pack(graphs)
    with _lib.engine(None) as eng:
        eng.pack(gp, rp, ci, ids, None, None)
        eng.sm_features(int(k.k), k.lambdas_, vt, et, elids, flags)
        return eng.sm_counts(n_fit, row)


def _record_words(n, elab):
    W = (n + 31) // 32
    return 2 * n * W + n + (n * n if elab else 0)


def _check_sm(X, Y, kk=5, counts=True, **kw):
    """K of fit_transform(X) and transform(Y) against sm_oracle.gram, and (counts) every pair's tv against
    sm_oracle.counts."""
    k = SubgraphMatching(k=kk, **kw)
    K = k.fit_transform(X)
    assert np.array_equal(K, sm_oracle.gram(k.X, None, k.kv, k.ke, kk, k.lambdas_))
    for row in range(len(X) if counts else 0):
        tv = _counts(k, k.X, len(X), row)
        for c in range(len(X)):
            x, y = (k.X[row], k.X[c]) if row <= c else (k.X[c], k.X[row])
            assert np.array_equal(tv[c], [float(t) for t in sm_oracle.counts(x, y, k.kv, k.ke, kk)]), (row, c)
    if Y is not None:
        Kt = k.transform(Y)
        assert np.array_equal(Kt, sm_oracle.gram(k.X, k.parse_input(Y), k.kv, k.ke, kk, k.lambdas_))
    return k


@pytest.mark.parametrize("variant", ["labelled", "ke_none", "directed"])
def test_sm_bench_graphs(variant):
    W = gen_workload(24)
    if variant == "directed":
        W = _directed(W, 9, 0.0)
    nmax = max(len(x[1]) for x in W)
    elab = variant != "ke_none"
    # 8 warps x two records of the largest pair in 96 KiB of shared memory, or read from global memory
    assert (8 * 2 * _record_words(nmax, elab) * 4 > 96 * 1024) == elab
    _check_sm(W[:20], W[20:], counts=variant == "labelled", **({} if elab else {"ke": None}))


def _with_hub(x, degree, seed, mixed=True):
    """x with a vertex 0 (the smallest id, so it roots the largest extension sets) joined to `degree` vertices, both
    ways or (mixed) out-edges to some, in-edges from others, both ways to the rest; the other vertices move up by
    one."""
    g, L = x[0], x[1]
    rng = np.random.default_rng(seed)
    e = {(u + 1, v + 1): 1 for (u, v) in g}
    L2 = {v + 1: l for v, l in L.items()}
    L2[0] = 0
    for i, v in enumerate(rng.choice(len(L), size=min(degree, len(L)), replace=False).tolist()):
        if not mixed or i % 3 != 1:
            e[(0, v + 1)] = 1
        if not mixed or i % 3 != 2:
            e[(v + 1, 0)] = 1
    return [e, L2, {(u, v): (L2[u] + L2[v]) % 3 for (u, v) in e}]


def test_sm_hub_labelled():
    """Bench graphs with a hub of in- and out-degree ~20 at k = 5 and 6: the stack bound 1 + sum d D^2 is large."""
    W = gen_workload(8)
    X = [_with_hub(W[0], 24, 1), W[1], _with_hub(W[2], 20, 2), W[3], W[4]]
    for kk in (5, 6):
        _check_sm(X, [W[5], _with_hub(W[6], 22, 3)], kk=kk)


def test_sm_hub_unlabelled_fills_the_stack():
    """kv = ke = None and a hub of degree D = 20 paired with itself at k = 3: the root (hub, hub) has D^2 extension
    candidates and its first child about (D - 1)^2 more, within the bound 1 + D^2 + 2 D^2 but past 1 + D^2."""
    W = gen_workload(4)
    X = [_with_hub(W[0], 20, 4, mixed=False), W[1]]
    _check_sm(X, None, kk=3, kv=None, ke=None)
