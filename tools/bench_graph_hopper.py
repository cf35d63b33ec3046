"""GraphHopper on config 5's graphs (2 000 ER graphs, avg 40 nodes, d = 16 attributes, seed 0): linear and gaussian.

Prints one JSON line: ms per pass split into node maps + feature map / self similarities (one features call) and the
Gram, delta and the feature dimension, node pairs/s, the node-pair Gram's fp64 FLOP/s against the H100 SXM data-sheet
peaks (34 TFLOP/s FP64 FMA, 67 TFLOP/s FP64 tensor core), the GPU name and power limit, and -- when oracle/_ref holds
the reference -- the reference's time on a bounded sample of connected graphs.

    python tools/bench_graph_hopper.py [--steps 5] [--warmup 2] [--ref-graphs 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

FP64_FMA_PEAK, FP64_DMMA_PEAK = 34.0, 67.0  # TFLOP/s, H100 SXM data sheet (700 W)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0] if q else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ref-graphs", type=int, default=20)
    args = ap.parse_args()
    from bench import gen_list
    from grakel_b200 import _lib
    from grakel_b200.packing import pack

    X = gen_list(2000, 40, 0, attr=16, as_adj=True)
    b = pack(X, "sp", need_labels=True, attributes=True, want_weights=True)
    n, V, d = b.n_graphs, b.n_vertices, b.attrs.shape[1]
    out = {"workload": "GraphHopper on config5's graphs: 2000 ER graphs (avg 40 nodes, d=16, seed 0)", "gpu": gpu_info(),
           "n_graphs": n, "n_vertices": V}
    eng = _lib.get_engine()
    eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, None, None, b.attrs)
    for name, nk, mu in (("linear", _lib.GK_GH_LINEAR, 1.0), ("gaussian", _lib.GK_GH_GAUSSIAN, 1.0)):
        feats, grams, totals = [], [], []
        for i in range(args.warmup + args.steps):
            t0 = time.perf_counter()
            st = eng.gh_features(nk, mu)
            eng.gram(n, out=False, stats=st, want_diag=False)
            t1 = time.perf_counter()
            if i >= args.warmup:
                feats.append(st.ms_features)
                grams.append(st.ms_gemm)
                totals.append((t1 - t0) * 1e3)
        delta = int(st.level_dims[0])
        T = delta * (delta + 1) // 2
        r = {"delta": delta, "map_row_length": T, "feature_dim": int(st.n_columns), "gram_path": int(st.gram_path),
             "ms_node_maps_plus_features": float(np.median(feats)), "ms_gram": float(np.median(grams)),
             "ms_per_pass_host": float(np.median(totals)),
             "graph_pairs_per_s": n * n / (np.median(totals) * 1e-3)}
        if name == "linear":
            fl = 2.0 * n * n * int(st.n_columns)
            r["gram_note"] = "3xTF32 or fp64 Gram of the ShortestPathAttr route; 2 N^2 D algorithmic flops"
        else:
            # upper triangle of the node-pair matrix: <M_v, M_v'> (2T flops) and ||x_v - x_v'||^2 (3d flops)
            fl = V * (V + 1) / 2.0 * (2.0 * T + 3.0 * d)
            r["node_pairs_per_s"] = V * (V + 1) / 2.0 / (np.median(grams) * 1e-3)
            r["gram_note"] = "fused fp64 CUDA-core node-pair Gram (FMA, no DMMA); upper tiles only"
        tfl = fl / (np.median(grams) * 1e-3) / 1e12
        r["gram_tflops"] = tfl
        if name != "linear":  # the linear Gram runs on the tf32 tensor cores (gram_path 4) or fp64 (5)
            r["frac_of_fp64_fma_peak"] = tfl / FP64_FMA_PEAK
            r["frac_of_fp64_dmma_peak"] = tfl / FP64_DMMA_PEAK
        out[name] = r
    ref_dir = os.path.join(ROOT, "oracle", "_ref")
    if os.path.isdir(os.path.join(ref_dir, "grakel")) and args.ref_graphs > 0:
        sys.path.insert(0, ref_dir)
        import warnings
        from grakel.kernels import GraphHopper as RefGH
        from make_golden_graph_hopper import connected
        from grakel_b200 import GraphHopper
        Xs = connected(args.ref_graphs, 40, 0, dim=16)  # connected: the reference raises on isolated vertices
        warnings.simplefilter("ignore")
        for kt in ("linear", "gaussian"):
            t0 = time.perf_counter()
            Kr = RefGH(kernel_type=kt).fit_transform(Xs)
            tr = time.perf_counter() - t0
            Kd = GraphHopper(kernel_type=kt).fit_transform(Xs)
            out["reference_" + kt] = {"graphs": len(Xs), "s": tr, "graph_pairs_per_s": len(Xs) ** 2 / tr,
                                      "max_rel_diff_vs_device": float(np.max(np.abs(Kd - Kr)) / np.max(np.abs(Kr)))}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
