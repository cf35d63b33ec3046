"""CoreFramework over NeighborhoodHash, OddSth, WeisfeilerLehmanOptimalAssignment and SubgraphMatching (ke=None):
fit_transform on bench.gen_list(2000, 40, 0) (edge labels added for SubgraphMatching, whose reference reads them),
split into host level construction (packing, core numbers, level blocks), the base kernels (their per-level label
parses on the host and feature passes on the device) and the fold (gk_core_level_add: each level's Gram and its
scatter, and the one fetch of K), beside the reference on the first `--ref-graphs` graphs,
extrapolated linearly to 2000 graphs: a lower bound, the per-level Grams being quadratic in the graph count.
Prints one JSON line per base, with the card and its power limit.

    python tools/bench_core_bases.py [--ref-graphs 40] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from grakel_b200 import (CoreFramework, NeighborhoodHash, OddSth, SubgraphMatching,  # noqa: E402
                         WeisfeilerLehmanOptimalAssignment)

BASES = {"NH": (NeighborhoodHash, {"random_state": 0}), "ODD": (OddSth, {}),
         "WL-OA": (WeisfeilerLehmanOptimalAssignment, {}), "SM": (SubgraphMatching, {"k": 3, "ke": None})}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        return "unknown"


def reference_seconds(name, G, n):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    try:
        from grakel import kernels as rk
    except ImportError:
        return None
    base, params = BASES[name]
    k = rk.CoreFramework(base_graph_kernel=(getattr(rk, base.__name__), dict(params)))
    t = time.perf_counter()
    k.fit_transform(G[:n])
    return time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref-graphs", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    gpu = card()
    G0 = bench.gen_list(2000, 40, 0)
    for name, (base, params) in BASES.items():
        G = [[g, L, {e: 1 for e in g}] for g, L in G0] if name == "SM" else G0
        k = CoreFramework(base_graph_kernel=(base, dict(params)))
        k.fit_transform(G[:50])  # warm-up: module load, buffers
        runs = []
        for _ in range(a.reps):
            t = time.perf_counter()
            k.fit_transform(G)
            runs.append((time.perf_counter() - t, dict(k.stage_times_)))
        best, st = min(runs, key=lambda r: r[0])
        ref = reference_seconds(name, G, a.ref_graphs)
        print(json.dumps({"base": name, "graphs": len(G), "levels": k._max_core_number + 1,
                          "fit_transform_s": round(best, 3),
                          "host_level_construction_s": round(st["levels"], 3),
                          "base_kernels_s": round(st["base"], 3), "fold_s": round(st["fold"], 3),
                          "reference_s_lower_bound": None if ref is None else round(ref * len(G) / a.ref_graphs, 1),
                          "reference_graphs_timed": a.ref_graphs, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
