"""Random walk kernels on the config-2 graph sizes: bench.gen_list(2000, 40, 0) with RandomWalk and RandomWalkLabeled,
fast/geometric (conjugate gradients per pair) and fast/exponential (spectral; RandomWalkLabeled: Taylor series).
Prints one JSON line: ms per pass split into host eigen work, device pair kernels and delivery, graph pairs/s, the
fp64 rate of the CG matvecs against the 34 TFLOP/s FP64 FMA data-sheet figure, the GPU and its power limit, and --
when oracle/_ref holds the reference -- its time on a 20-graph sample and the largest relative difference there.

    python tools/bench_random_walk.py [--graphs 2000] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP64_PEAK = 34e12  # H100 SXM data sheet, FP64 (non-tensor) FMA rate


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [x.strip() for x in out.split(",")]
    except Exception:
        return None


def cg_flops(est, X, its):
    """fp64 FLOP of the CG matvecs as the unmasked edge-pair product counts them: per iteration and entry of the pair
    grid, 2 per (out-edge of u, in-edge of u') pair plus 3 for q = p - lamda y; symmetric pairs counted once."""
    m = np.array([np.count_nonzero(A) for A in est.X.mats], dtype=np.float64)
    n = np.array([A.shape[0] for A in est.X.mats], dtype=np.float64)
    iu = np.triu_indices(len(m))
    per_it = 2.0 * np.outer(m, m) + 3.0 * np.outer(n, n)
    return float(np.sum(its[iu].astype(np.float64) * per_it[iu]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import bench
    from grakel_b200 import RandomWalk, RandomWalkLabeled, _lib
    X = bench.gen_list(a.graphs, 40, 0)
    n = len(X)
    pairs = n * (n + 1) // 2
    res = {"workload": "gen_list(%d, 40, 0)" % n, "pairs": pairs, "gpu": gpu_info(), "runs": {}}
    warnings.simplefilter("ignore")
    for cls in (RandomWalk, RandomWalkLabeled):
        for kt in ("geometric", "exponential"):
            est = cls(lamda=0.01, kernel_type=kt)
            est.fit_transform(X)  # warm-up
            wall, dev, eig, d2h = [], [], [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                K = est.fit_transform(X)
                wall.append((time.perf_counter() - t0) * 1e3)
                dev.append(est.stats_.ms_rw)
                d2h.append(est.stats_.ms_d2h)
                eig.append(est.ms_host_eig_)
            r = {"ms_pass": min(wall), "ms_host_eig": min(eig), "ms_device": min(dev), "ms_delivery": min(d2h),
                 "pairs_per_s": pairs / (min(wall) * 1e-3), "gram_path": int(est.stats_.gram_path)}
            if est.stats_.gram_path == 8 and cls is RandomWalk:
                its = _lib.get_engine().rw_iterations(n, n)
                fl = cg_flops(est, X, its)
                r.update(cg_flop=fl, cg_flops_per_s=fl / (min(dev) * 1e-3),
                         cg_frac_fp64_peak=fl / (min(dev) * 1e-3) / FP64_PEAK, mean_cg_iterations=float(its.mean()))
            ref_dir = os.path.join(ROOT, "oracle", "_ref")
            if os.path.isdir(os.path.join(ref_dir, "grakel")):
                sys.path.insert(0, ref_dir)
                import grakel.kernels as gk
                ref = getattr(gk, cls.__name__)(lamda=0.01, kernel_type=kt)
                t0 = time.perf_counter()
                Kr = ref.fit_transform(X[:20])
                r["ref_ms_20_graphs"] = (time.perf_counter() - t0) * 1e3
                r["ref_ms_per_pair"] = r["ref_ms_20_graphs"] / 210
                Ks = cls(lamda=0.01, kernel_type=kt).fit_transform(X[:20])
                r["max_rel_diff_20_graphs"] = float(np.max(np.abs(Ks - Kr) / np.maximum(np.abs(Kr), 1e-300)))
            res["runs"]["%s/%s" % (cls.__name__, kt)] = r
            del K
    print(json.dumps(res))


if __name__ == "__main__":
    main()
