"""SubgraphMatching device time at k = 5 on two workloads, and the real reference (oracle/_ref) on the host.

    python tools/bench_subgraph_matching.py [--n 2000] [--repeat 3] [--ref-pairs 200] [--out result.json]

Workloads: the bundled MUTAG (188 graphs, node and edge labels, the dirac defaults), and bench.gen_list(n, 40, 0)
with ke=None (the generator has no edge labels).  One pass is the fit_transform Gram: the self similarities and the
upper triangle, N (N + 1) / 2 + N pair evaluations (ms_rw of gk_gram, CUDA events; median of `repeat` passes after
a warm-up pass).  With the uniform lambdas and integer weights K[i, j] = sum(tv) counts the connected cliques of the
pair, so the clique total of a pass is the sum of K's upper triangle plus the diagonal once more.  The reference is
timed on its own pairwise_operation over `ref-pairs` pairs spread over the triangle and extrapolated to the pass.
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
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def reference_time(X, params, n_pairs, n_eval):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "grakel")):
        return None
    sys.path.insert(0, ref)
    from grakel.kernels import SubgraphMatching as Ref
    k = Ref(**params)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        k.fit(X)
    rng = np.random.default_rng(0)
    N = len(k.X)
    pairs = [tuple(sorted(rng.integers(0, N, 2))) for _ in range(n_pairs)]
    t0 = time.perf_counter()
    for i, j in pairs:
        k.pairwise_operation(k.X[i], k.X[j])
    dt = time.perf_counter() - t0
    return {"pairs": n_pairs, "seconds": dt, "ms_per_pair": dt * 1e3 / n_pairs,
            "extrapolated_pass_s": dt / n_pairs * n_eval}


def run(name, X, params, repeat, ref_pairs):
    from grakel_b200 import SubgraphMatching, _lib
    k = SubgraphMatching(**params).fit(X)
    gp, rp, ci, ids, elids, vt, et, flags = k._pack(k.X)
    N = len(X)
    n_eval = N * (N + 1) // 2 + N
    times = []
    with _lib.engine() as eng:
        eng.pack(gp, rp, ci, ids, None, None)
        for it in range(repeat + 1):
            t0 = time.perf_counter()
            st = eng.sm_features(int(k.k), k.lambdas_, vt, et, elids, flags)
            K, xd, _ = eng.gram(N, stats=st)
            wall = (time.perf_counter() - t0) * 1e3
            if it:
                times.append({"pairs": st.ms_rw, "d2h": st.ms_d2h, "wall": wall})
    med = {key: float(np.median([t[key] for t in times])) for key in times[0]}
    cliques = float(np.sum(np.triu(K))) + float(np.sum(xd))
    s = med["pairs"] * 1e-3
    out = {"workload": name, "graphs": N, "pair_evaluations": n_eval, "median_ms": med,
           "pairs_per_s": n_eval / s, "cliques": cliques, "cliques_per_s": cliques / s,
           "reference_host": reference_time(X, params, ref_pairs, n_eval)}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--ref-pairs", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from bench import gen_list
    from nspd_cases import mutag
    result = {"card": card(), "runs": []}
    result["runs"].append(run("MUTAG, k = 5", mutag(), dict(k=5), a.repeat, a.ref_pairs))
    gen = [[g, L, {}] for g, L in gen_list(a.n, 40, 0)]
    result["runs"].append(run("bench.gen_list(%d, 40, 0), ke = None, k = 5" % a.n, gen, dict(k=5, ke=None), a.repeat,
                              a.ref_pairs))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
