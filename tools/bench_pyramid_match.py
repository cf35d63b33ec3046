"""PyramidMatch and WeisfeilerLehman over PyramidMatch, stage by stage: the host embedding (scipy eigs / numpy eig, one
call per graph and embedding set), the device stages (cells + per-level columns, per-level integer Grams, combine),
the fp64 delivery and end to end; the reference (oracle/_ref) on a subset, extrapolated by N^2.  Prints one JSON line
per run; report the card name and power limit beside the numbers.

    python tools/bench_pyramid_match.py [--n 10000] [--n-wl 2000] [--runs 3] [--ref-n 150]
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

import bench  # noqa: E402
from grakel_b200 import PyramidMatch, WeisfeilerLehman  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception:  # noqa: BLE001
        return "unknown"


def stages(est, t_e2e):
    st = est.stats_
    return {"host_embed_ms": round(est.ms_host_embed_, 1), "columns_ms": round(st.ms_columns, 2),
            "level_gram_ms": round(st.ms_gemm, 2), "combine_ms": round(st.ms_combine, 2),
            "d2h_ms": round(st.ms_d2h, 2), "e2e_ms": round(t_e2e * 1e3, 1)}


def run_pm(X):
    est = PyramidMatch(L=4, d=6)
    t0 = time.perf_counter()
    est.fit_transform(X)
    return stages(est, time.perf_counter() - t0)


def run_wl(X, h):
    est = WeisfeilerLehman(n_iter=h, base_graph_kernel=PyramidMatch)
    t0 = time.perf_counter()
    est.fit_transform(X)
    return stages(est, time.perf_counter() - t0)


def run_ref(X, N, wl_h=None):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel.kernels import PyramidMatch as RefPM, WeisfeilerLehman as RefWL
    est = RefPM(L=4, d=6) if wl_h is None else RefWL(n_iter=wl_h, base_graph_kernel=RefPM)
    t0 = time.perf_counter()
    est.fit_transform(X)
    t = time.perf_counter() - t0
    return {"ref_n": len(X), "ref_s": round(t, 2), "ref_extrapolated_s": round(t * (N / len(X)) ** 2, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--n-wl", type=int, default=2000)
    ap.add_argument("--wl-iter", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--ref-n", type=int, default=150)
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    X = bench.gen_list(a.n, 40, 0)
    Xw = X[:a.n_wl]
    gpu = card()
    run_pm(X[:200])  # warm-up: library load, engine, allocations
    for r in range(a.runs):
        print(json.dumps({"kernel": "PM", "run": r, "n": a.n, "gpu": gpu, **run_pm(X)}), flush=True)
        print(json.dumps({"kernel": "WL-PM", "run": r, "n": a.n_wl, "h": a.wl_iter, "gpu": gpu,
                          **run_wl(Xw, a.wl_iter)}), flush=True)
    if a.ref_n > 0 and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "grakel")):
        print(json.dumps({"kernel": "PM", "reference": True, **run_ref(X[:a.ref_n], a.n)}), flush=True)
        print(json.dumps({"kernel": "WL-PM", "reference": True,
                          **run_ref(Xw[:max(a.ref_n // 3, 10)], a.n_wl, wl_h=a.wl_iter)}), flush=True)


if __name__ == "__main__":
    main()
