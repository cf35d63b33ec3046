"""HadamardCode over SubgraphMatching, PyramidMatch and NeighborhoodSubgraphPairwiseDistance: fit_transform end to end
(host parsing and the fp64 delivery included, the host clock around work that ends in a device synchronise) on
bench.gen_list(2000, 40, 0) with edge labels (L_u + L_v) % 3, median of --runs after one warm-up run; for
SubgraphMatching also the per-level device route (n_iter SubgraphMatching runs on the level's Hadamard-code classes,
summed in level order).  With --ref, the reference (oracle/_ref) on the first 40 graphs, extrapolated linearly to 2000
graphs: a lower bound, since its pair work grows with N^2.  Prints one JSON line per run with the card name and power
limit, read in the same process.

    python tools/bench_hc_bases.py [--runs 3] [--n-iter 5] [--bases SM,PM,NSPD] [--ref]
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

import bench  # noqa: E402
from grakel_b200 import HadamardCode, NeighborhoodSubgraphPairwiseDistance, PyramidMatch, SubgraphMatching  # noqa: E402

BASES = {"SM3": (SubgraphMatching, {"k": 3}), "SM5": (SubgraphMatching, {"k": 5}),
         "PM": (PyramidMatch, {}), "NSPD": (NeighborhoodSubgraphPairwiseDistance, {})}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        return "unknown"


def workload(n):
    return [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in bench.gen_list(n, 40, 0)]


def timed(fn, runs):
    fn()  # warm-up: engine set-up, first launches
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def per_level(X, n_iter, params):
    import hc_bases_oracle
    import hc_oracle
    enum = hc_oracle.enumerate_labels([x[1] for x in X])
    levels = hc_bases_oracle.level_elements(X, n_iter, enum)  # host relabel, outside the timed part

    def run():
        return np.sum([SubgraphMatching(**params).fit_transform(lx) for lx in levels], axis=0)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--n-iter", type=int, default=5)
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--bases", default="SM3,SM5,PM,NSPD")
    ap.add_argument("--ref", action="store_true")
    a = ap.parse_args()
    X = workload(a.n)
    gpu = card()
    for name in a.bases.split(","):
        base, params = BASES[name]
        out = {"bench": "hc_bases", "base": name, "params": params, "n_iter": a.n_iter, "n_graphs": a.n, "gpu": gpu}
        out["fit_transform_s"] = round(timed(lambda: HadamardCode(n_iter=a.n_iter, base_graph_kernel=(base, dict(
            params))).fit_transform(X), a.runs), 3)
        if base is SubgraphMatching:
            out["per_level_device_s"] = round(timed(per_level(X, a.n_iter, params), a.runs), 3)
        if a.ref:
            sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
            import grakel.kernels as ref
            rb = getattr(ref, base.__name__)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                t0 = time.perf_counter()
                ref.HadamardCode(n_iter=a.n_iter, base_graph_kernel=(rb, dict(params))).fit_transform(X[:40])
                t = time.perf_counter() - t0
            out["ref_40_s"] = round(t, 2)
            out["ref_lower_bound_s"] = round(t * a.n / 40, 1)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
