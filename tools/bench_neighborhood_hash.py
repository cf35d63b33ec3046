"""NeighborhoodHash stage times on config 2's graphs (10 000 ER graphs, mean 40 vertices, 7 labels, seed 0), R = 3,
both nh_type values, bits = 8 and 16, each stage against a byte floor; the real reference (oracle/_ref) on the host
for a prefix, extrapolated to the whole set with pairs/s held constant.

    python tools/bench_neighborhood_hash.py [--n 10000] [--repeat 5] [--ref-prefix 150] [--out result.json]

Stages (CUDA events of the library): hash (R levels of gk_nh_features), columns (per-level code compaction, counts,
unary expansion), the exact integer Gram of every level, the fp64 combine, the D2H copy of K.  Floors are HBM bytes at
the data-sheet 3.35 TB/s; they are estimates of the least traffic, not measurements:
  hash      R (V codes + V flags read, E neighbour codes and flags read, V codes + flags written)
  columns   R (V codes + flags read, V table probes, V count-table updates, V expanded entries written)
  gram      one fp32 N x N count matrix written (its upper triangle read back by the combine is counted there)
  combine   R fp32 upper triangles read + one fp64 N x N written: (2R + 8) N^2 bytes
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

HBM = 3.35e12


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def floors(N, V, E, R):
    return {
        "hash": R * (9 * V + 9 * E + 9 * V) / HBM * 1e3,
        "columns": R * (9 * V + 3 * 16 * V + 12 * V) / HBM * 1e3,
        "gram_per_level": 4.0 * N * N / HBM * 1e3,
        "combine": (2 * R + 8) * N * N / HBM * 1e3,
    }


def reference_time(X, R, nh_type, bits, prefix):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "grakel")):
        return None
    sys.path.insert(0, ref)
    from grakel.kernels import NeighborhoodHash as RefNH
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        RefNH(R=R, nh_type=nh_type, bits=bits, random_state=0).fit_transform(X[:prefix])
    dt = time.perf_counter() - t0
    pairs = prefix * (prefix + 1) / 2
    full = len(X) * (len(X) + 1) / 2
    return {"prefix": prefix, "seconds": dt, "pairs_per_s": pairs / dt, "extrapolated_s": full / (pairs / dt)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10000)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--ref-prefix", type=int, default=150)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from grakel_b200 import NeighborhoodHash, _lib
    from oracle.gk_oracle import gen

    X = gen(a.n, 40, 0)
    R = 3
    result = {"card": card(), "workload": "config2 graphs: %d ER graphs, mean 40 vertices, 7 labels, seed 0; R = 3" % a.n,
              "runs": []}
    for nh_type in ("simple", "count_sensitive"):
        for bits in (8, 16):
            nh = NeighborhoodHash(R=R, nh_type=nh_type, bits=bits, random_state=0).fit(X)
            F = nh.X
            b = F.block
            times = []
            with _lib.engine() as eng:
                eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, F.ids, None, None)
                for it in range(a.repeat + 1):
                    t0 = time.perf_counter()
                    st = eng.nh_features(R, nh._nh_code, bits, F.codes, F.valid)
                    K, _, _ = eng.gram(b.n_graphs, stats=st, want_diag=False)
                    wall = (time.perf_counter() - t0) * 1e3
                    if it:  # the first pass warms every shape
                        times.append({"hash": st.ms_hash, "columns": st.ms_columns,
                                      "gram_levels": list(st.ms_level_gram)[:R], "combine": st.ms_combine,
                                      "d2h": st.ms_d2h, "wall": wall})
            med = {k: float(np.median([t[k] for t in times])) for k in ("hash", "columns", "combine", "d2h", "wall")}
            med["gram_levels"] = [float(np.median([t["gram_levels"][r] for t in times])) for r in range(R)]
            fl = floors(b.n_graphs, b.n_vertices, len(b.col_idx), R)
            run = {"nh_type": nh_type, "bits": bits, "median_ms": med, "floor_ms": fl,
                   "floor_over_time": {"hash": fl["hash"] / med["hash"], "columns": fl["columns"] / med["columns"],
                                       "gram": [fl["gram_per_level"] / g for g in med["gram_levels"]],
                                       "combine": fl["combine"] / med["combine"]},
                   "level_dims": list(st.level_dims)[:R], "K_checksum": float(np.sum(K))}
            run["reference_host"] = reference_time(X, R, nh_type, bits, a.ref_prefix)
            result["runs"].append(run)
            print(json.dumps(run), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
