"""HadamardCode over VertexHistogram and over ShortestPath, stage by stage: the relabel (vectors, classes, VH counts),
columns + panel and the Gram from gk_stats; the device-resident pass (pack -> features -> Gram, K left on the device)
and end to end (host parsing and the fp64 delivery included); the relabel's algorithmic bytes,
V * W * 8 * (2 + mean out-degree) per level, over its time against the 3.35 TB/s of HBM3; the reference (oracle/_ref)
on 200 and 1 000 graphs, extrapolated by N^2.  Prints one JSON line per run; the card name and power limit are read
in the same process.

    python tools/bench_hadamard_code.py [--runs 3] [--n-sp 5000] [--ref]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import warnings


ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from grakel_b200 import HadamardCode, ShortestPath, _lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # noqa: BLE001
        return "unknown"


def device_pass(est, n_iter, sp):
    """pack -> gk_hc_features -> gk_gram with K left on the device, timed with CUDA events on the engine's stream."""
    data = est.X
    block = data.block
    with _lib.engine() as eng:
        eng.event_record(0)
        eng.pack(block.graph_ptr, block.row_ptr, block.col_idx, data.ids, block.weights if sp else None, None)
        st = eng.hc_features(n_iter, est._width, skip=None if sp else data.skip, sp=sp,
                             dijkstra_order=est._dijkstra_order(block) if sp else False)
        eng.gram(block.n_graphs, out=False, want_diag=False, stats=st)
        eng.event_record(1)
        eng.sync()
        ms = eng.event_elapsed(0, 1)
    return st, ms


def run(X, n_iter, sp):
    est = HadamardCode(n_iter=n_iter, base_graph_kernel=(ShortestPath, {}) if sp else None)
    t0 = time.perf_counter()
    est.fit_transform(X)
    e2e = time.perf_counter() - t0
    st, ms = device_pass(est, n_iter, sp)
    block = est.X.block
    V, E = block.n_vertices, len(block.col_idx)
    relabel_bytes = V * est._width * 8 * (2 + E / V) * n_iter
    return {"V": V, "E": E, "W": est._width, "relabel_ms": round(st.ms_hash, 3),
            "columns_panel_ms": round(st.ms_panel, 3), "gram_ms": round(st.ms_gemm + st.ms_tail, 3),
            "sp_features_ms": round(st.ms_features, 3) if sp else None,
            "hash_retries": int(st.hash_retries), "device_pass_ms": round(ms, 3), "e2e_ms": round(e2e * 1e3, 1),
            "relabel_GBps": round(relabel_bytes / (st.ms_hash * 1e-3) / 1e9, 1),
            "relabel_frac_hbm": round(relabel_bytes / (st.ms_hash * 1e-3) / HBM_BYTES_PER_S, 3)}


def run_ref(X, N, n_iter, sp):
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel.kernels import HadamardCode as RefHC, ShortestPath as RefSP
    est = RefHC(n_iter=n_iter, base_graph_kernel=RefSP if sp else None)
    t0 = time.perf_counter()
    est.fit_transform(X)
    t = time.perf_counter() - t0
    return {"ref_n": len(X), "ref_s": round(t, 3), "ref_extrapolated_s": round(t * (N / len(X)) ** 2, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--n-sp", type=int, default=5000, help="graphs of the HC-SP workload")
    ap.add_argument("--ref", action="store_true", help="also time the reference on 200 and 1 000 graphs")
    a = ap.parse_args()
    warnings.simplefilter("ignore")
    Xv = bench.gen_list(10000, 40, 0)
    Xs_all = bench.gen_list(5000, 60, 0, as_adj=True)
    Xs = Xs_all[:a.n_sp]
    gpu = card()
    run(Xv[:200], 5, False)  # warm-up: library load, engine, allocations
    run(Xs[:200], 3, True)
    for r in range(a.runs):
        print(json.dumps({"kernel": "HC-VH", "run": r, "n": len(Xv), "n_iter": 5, "gpu": gpu, **run(Xv, 5, False)}),
              flush=True)
        print(json.dumps({"kernel": "HC-SP", "run": r, "n": len(Xs), "n_iter": 3, "gpu": gpu, **run(Xs, 3, True)}),
              flush=True)
    if a.ref and os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "grakel")):
        for n in (200, 1000):
            print(json.dumps({"kernel": "HC-VH", "reference": True, **run_ref(Xv[:n], len(Xv), 5, False)}), flush=True)
            print(json.dumps({"kernel": "HC-SP", "reference": True, **run_ref(Xs_all[:n], len(Xs_all), 3, True)}), flush=True)


if __name__ == "__main__":
    main()
