"""Stage times of SvmTheta on the device, from the stats of its C-ABI stages, and the reference's host time on a sample
of the same graphs.

    python tools/bench_svm_theta.py [--graphs 2000 10000] [--ref-graphs 100] [--out results/svmt_bench.json]

Workloads: bench.gen_list(G, 40, 0, as_adj=True) (20 to 60 vertices) for every G of --graphs, at the default
subsets_size_range (2, 8) and at (6, 8).  The reference runs on the first --ref-graphs graphs of the first workload
when oracle/_ref is installed; its per-graph work (eigenvalue, SVM, draws) grows with the number of graphs and its
Gram with N^2, so its time is extrapolated as t_parse * (G / g) + t_gram * (G / g)^2 with both parts measured, and
labelled so."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from grakel_b200 import SvmTheta, _lib  # noqa: E402


def device_run(X, rng, reps=3):
    best = None
    for _ in range(reps):
        k = SvmTheta(random_state=0, subsets_size_range=rng)
        t0 = time.perf_counter()
        k.fit_transform(X)
        wall = (time.perf_counter() - t0) * 1e3
        s = k.svmt_stats_
        stages = {key: s[key] for key in ("h2d_ms", "eigenvalue_ms", "smo_ms", "host_draw_ms", "phi_ms", "d2h_ms")}
        stages["fit_transform_wall_ms"] = wall
        if best is None or wall < best["fit_transform_wall_ms"]:
            best = stages
    k = SvmTheta(random_state=0, subsets_size_range=rng)
    k.initialize()
    with _lib.engine() as eng:
        k._svmt_run(eng, X)
        eng.gram(len(X))  # warm
        st = _lib.GkStats()
        eng.gram(len(X), stats=st)
    best["gram_ms"] = st.ms_gemm
    best["gram_d2h_ms"] = st.ms_d2h
    best["gram_path"] = st.gram_path
    best["n_graphs"] = len(X)
    return best


def reference_run(X, g):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel.kernels import SvmTheta as Ref
    k = Ref(random_state=0)
    t0 = time.perf_counter()
    k.fit(X[:g])
    t_parse = time.perf_counter() - t0
    t0 = time.perf_counter()
    k._calculate_kernel_matrix()
    t_gram = time.perf_counter() - t0
    return t_parse, t_gram


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, nargs="+", default=[2000, 10000])
    ap.add_argument("--ref-graphs", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu}
    for G in a.graphs:
        X = bench.gen_list(G, 40, 0, as_adj=True)
        for rng in ((2, 8), (6, 8)):
            res["gen_list_%d_range_%d_%d" % (G, *rng)] = device_run(X, rng)
    if os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "grakel")) and a.ref_graphs > 0:
        X = bench.gen_list(a.graphs[0], 40, 0, as_adj=True)
        t_parse, t_gram = reference_run(X, a.ref_graphs)
        for G in a.graphs:
            r = G / a.ref_graphs
            res["reference_%d" % G] = {"graphs_timed": a.ref_graphs, "parse_s": t_parse, "gram_s": t_gram,
                                       "extrapolated_s": t_parse * r + t_gram * r * r, "extrapolated": True}
    print(json.dumps(res, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
