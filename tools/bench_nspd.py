"""NeighborhoodSubgraphPairwiseDistance stage times at the defaults (r = 3, d = 4) on two workloads, and the real
reference (oracle/_ref) on the host.

    python tools/bench_nspd.py [--n 2000] [--repeat 5] [--ref-prefix 40] [--out result.json]

Workloads: the bundled MUTAG (188 graphs, node and edge labels), and bench.gen_list(n, 40, 0) with edge label
(l_u + l_v) % 3.  Stages (CUDA events of the library, medians of `repeat` passes after one warm-up pass): BFS levels +
hashes (gk_nspd_features' ms_hash), columns (pairs, keys, per-level numbering and counts), the exact integer Gram of
every level (summed), the fp64 fold, the D2H copy of K; `wall` is the host time of features + Gram.
The reference is timed in full on MUTAG and on the first `ref-prefix` generator graphs; its extrapolation to the whole
set assumes its time is linear in the number of graphs (the per-graph parsing, hashing and counting; the sparse
per-level Grams are taken as negligible, which makes the extrapolation a lower bound).
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def gen_workload(n):
    from bench import gen_list
    out = []
    for g, L in gen_list(n, 40, 0):
        out.append([g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}])
    return out


def reference_time(X, prefix):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "grakel")):
        return None
    sys.path.insert(0, ref)
    from grakel.kernels import NeighborhoodSubgraphPairwiseDistance as Ref
    prefix = min(prefix, len(X))
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        Ref().fit_transform(X[:prefix])
    dt = time.perf_counter() - t0
    return {"graphs": prefix, "seconds": dt, "extrapolated_s_linear_in_graphs": dt * len(X) / prefix}


def run(name, X, repeat, ref_prefix):
    from grakel_b200 import NeighborhoodSubgraphPairwiseDistance, _lib
    k = NeighborhoodSubgraphPairwiseDistance().fit(X)
    gp, rp, ci, lab, el, sh, tokens = k._pack(k.X)
    N = len(X)
    times = []
    with _lib.engine() as eng:
        eng.pack(gp, rp, ci, lab, None, None)
        for it in range(repeat + 1):
            t0 = time.perf_counter()
            st, _ = eng.nspd_features(k.r, k.d, sh, el, tokens)
            fs = (st.ms_hash, st.ms_columns)
            K, _, _ = eng.gram(N, stats=st, want_diag=False)
            wall = (time.perf_counter() - t0) * 1e3
            if it:
                times.append({"bfs+hash": fs[0], "columns": fs[1], "gram_levels": float(sum(st.ms_level_gram)),
                              "fold": st.ms_combine, "d2h": st.ms_d2h, "wall": wall})
    med = {key: float(np.median([t[key] for t in times])) for key in times[0]}
    out = {"workload": name, "graphs": N, "vertices": int(gp[-1]), "directed_edges": int(len(ci)),
           "levels": int(st.n_levels), "columns": int(st.n_columns), "median_ms": med,
           "K_checksum": float(np.sum(K)), "reference_host": reference_time(X, ref_prefix)}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--ref-prefix", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from nspd_cases import mutag
    result = {"card": card(), "runs": []}
    M = mutag()
    result["runs"].append(run("MUTAG, r = 3, d = 4", M, a.repeat, len(M)))
    result["runs"].append(run("bench.gen_list(%d, 40, 0), edge label (l_u + l_v) %% 3, r = 3, d = 4" % a.n,
                              gen_workload(a.n), a.repeat, a.ref_prefix))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
