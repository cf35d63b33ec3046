"""Stage times of GraphletSampling's sampled route on the device, and the reference's host time on a few of the same
graphs.

    python tools/bench_graphlet_sampling.py [--graphs 2000 10000] [--ref-graphs 3] [--out results/gs_bench.json]

Workloads: bench.gen_list(G, 40, 0) (undirected, 20 to 60 vertices) for every G of --graphs, at k = 5 with
sampling {"epsilon": 0.05} (the reference's default bound: 5 617 samples per graph) and {"n_samples": 100}.  The
stages are the estimator's gs_stats_: the host MT19937 draws, the class table, the sample upload, the classification
and counting, the columns, and the Gram with its copy to the host.  The reference's time per graph is measured on the
first --ref-graphs graphs (its bins grow with the graphs, so the extrapolation to G graphs is a lower bound) and
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
from grakel_b200 import GraphletSampling  # noqa: E402

SAMPLINGS = [{"epsilon": 0.05}, {"n_samples": 100}]


def device_run(X, sampling, reps=2):
    best = None
    for _ in range(reps):
        k = GraphletSampling(k=5, sampling=dict(sampling), random_state=0)
        t0 = time.perf_counter()
        k.fit_transform(X)
        wall = (time.perf_counter() - t0) * 1e3
        s = dict(k.gs_stats_, fit_transform_wall_ms=wall)
        if best is None or wall < best["fit_transform_wall_ms"]:
            best = s
    return best


def reference_ms_per_graph(X, sampling, g):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel.kernels import GraphletSampling as Ref
    t0 = time.perf_counter()
    Ref(k=5, sampling=dict(sampling), random_state=0).fit_transform(X[:g])
    return (time.perf_counter() - t0) * 1e3 / g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, nargs="+", default=[2000, 10000])
    ap.add_argument("--ref-graphs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"card": card, "runs": []}
    print("card:", card)
    for G in a.graphs:
        X = bench.gen_list(G, 40, 0)
        for sampling in SAMPLINGS:
            device_run(X[:50], sampling, reps=1)  # warm: module load, class table
            r = dict(device_run(X, sampling), graphs=G, sampling=sampling)
            res["runs"].append(r)
            print(json.dumps(r))
    if a.ref_graphs and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "grakel")):
        X = bench.gen_list(a.ref_graphs, 40, 0)
        for sampling in SAMPLINGS:
            ms = reference_ms_per_graph(X, sampling, a.ref_graphs)
            r = {"reference_ms_per_graph": ms, "sampling": sampling, "measured_on_graphs": a.ref_graphs,
                 "extrapolated_lower_bound_s": {G: ms * G / 1e3 for G in a.graphs}}
            res["reference"] = res.get("reference", []) + [r]
            print(json.dumps(r))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
