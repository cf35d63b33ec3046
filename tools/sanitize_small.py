"""Small end-to-end calls of every device path for compute-sanitizer (memcheck / racecheck): WL (fused persistent
kernel, cooperative launch, grid barrier, CAS tables), head/tail Gram (wgmma + TMA + atomics), SP (bitmask BFS,
Floyd-Warshall, Dijkstra order), SP-attr (tf32 GEMM), WL-OA, transform (rectangular)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from bench import gen_list  # noqa: E402
from grakel_b200 import (ShortestPath, ShortestPathAttr, WeisfeilerLehman,  # noqa: E402
                         WeisfeilerLehmanOptimalAssignment)
from make_golden_dijkstra import gen_real  # noqa: E402

X = gen_list(300, 14, 3)
K = WeisfeilerLehman(n_iter=3).fit_transform(X)
Kn = WeisfeilerLehman(n_iter=3, normalize=True).fit(X[:250]).transform(X[250:])
print("WL", K.shape, float(K.sum()), Kn.shape)
os.environ["GRAKEL_B200_FORCE_T"] = "4"
K2 = WeisfeilerLehman(n_iter=3).fit_transform(X)
assert np.array_equal(K, K2)
del os.environ["GRAKEL_B200_FORCE_T"]
Ko = WeisfeilerLehmanOptimalAssignment(n_iter=2).fit_transform(X[:120])
print("WL-OA", Ko.shape, float(Ko.sum()))
A = gen_list(120, 16, 4, as_adj=True)
Ks = ShortestPath().fit_transform(A)
print("SP", Ks.shape, float(Ks.sum()))
R = gen_real(40, 10, 2)
Kr = ShortestPath().fit_transform(R)
Kf = ShortestPath(algorithm_type="floyd_warshall").fit_transform(R)
print("SP real", float(Kr.sum()), float(Kf.sum()))
At = gen_list(60, 12, 5, attr=4, as_adj=True)
Ka = ShortestPathAttr().fit_transform(At)
print("SP-attr", Ka.shape, float(Ka.sum()))
# the asynchronous pass (gk_wl_gram): first call synchronous (capacities), the next ones asynchronous
from grakel_b200 import _lib  # noqa: E402
from grakel_b200.packing import label_ids, pack  # noqa: E402
b = pack(X, "wl")
ids, _ = label_ids(b.labels, None, sort_new=False)
eng = _lib.Engine(0)
eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, ids)
for rep in range(3):
    Kg, _, st = eng.wl_gram(3)
    assert np.array_equal(Kg, K), rep
print("gk_wl_gram", Kg.shape, float(Kg.sum()), "asynchronous pass" if st.gemm_launches == 0 else "synchronous route")
# a user metric: device APSP + host contraction
Km = ShortestPathAttr(metric=lambda a, c: float(np.exp(-np.sum((np.asarray(a) - np.asarray(c)) ** 2)))).fit_transform(At[:8])
print("SP-attr metric", Km.shape, float(Km.sum()))
print("sanitize_small ok")
# WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance (per-level fold, device-resident level sum) and over OddSth
# (one DAG pass over all levels), fit_transform and a normalised transform
from grakel_b200 import NeighborhoodSubgraphPairwiseDistance, OddSth  # noqa: E402
Xe = [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in gen_list(40, 10, 6)]
for base in ((NeighborhoodSubgraphPairwiseDistance, {"r": 1, "d": 2}), (OddSth, {"h": 2})):
    wlb = WeisfeilerLehman(n_iter=2, normalize=True, base_graph_kernel=base)
    Kb = wlb.fit_transform(Xe[:30])
    Kt = wlb.transform(Xe[30:])
    print("WL over", base[0].__name__, Kb.shape, float(Kb.sum()), Kt.shape)
# CoreFramework over the fold bases (per-level Grams scattered into a device-resident sum), fit_transform and a
# normalised transform
from grakel_b200 import (CoreFramework, NeighborhoodHash, SubgraphMatching,  # noqa: E402
                         WeisfeilerLehmanOptimalAssignment)
for base in ((NeighborhoodHash, {"random_state": 0}), (OddSth, {}), (WeisfeilerLehmanOptimalAssignment, {}),
             (SubgraphMatching, {"k": 3, "ke": None})):
    cf = CoreFramework(normalize=base[0] is not OddSth, base_graph_kernel=base)
    Kc = cf.fit_transform(Xe[:30])
    Kt = cf.transform(Xe[30:])
    print("CORE over", base[0].__name__, Kc.shape, float(Kc.sum()), Kt.shape)
