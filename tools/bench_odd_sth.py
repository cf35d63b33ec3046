"""OddSth stage times at h = None and h = 3 on two workloads, and the real reference (oracle/_ref) on the host.

    python tools/bench_odd_sth.py [--n 2000] [--repeat 5] [--ref-prefix 40] [--out result.json]

Workloads: the bundled MUTAG (188 graphs, edges listed in sorted order), and bench.gen_list(n, 40, 0).  Stages (CUDA
events of the library, medians of `repeat` passes after one warm-up pass): DAGs and identities (gk_odd_features'
ms_hash: BFS, Kahn order, hashes, interning and verification), columns (numbering, C, phi, self similarities and the
bit-plane tables), the exact integer Gram of every bit plane with the fp64 fold, the D2H copy of K; `wall` is the host
time of features + Gram.  The reference is timed in full on MUTAG and on the first `ref-prefix` generator graphs; its
cost grows faster than linearly in the number of graphs (big_dag_append extends every feature's frequency list for
each new graph), so the linear extrapolation to the whole set is a lower bound.
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
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                                        "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def reference_time(X, prefix, h):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "grakel")):
        return None
    sys.path.insert(0, ref)
    from grakel.kernels import OddSth as Ref
    prefix = min(prefix, len(X))
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        Ref(h=h).fit_transform(X[:prefix])
    dt = time.perf_counter() - t0
    return {"graphs": prefix, "seconds": dt, "lower_bound_s_linear_in_graphs": dt * len(X) / prefix}


def run(name, X, h, repeat, ref_prefix):
    from grakel_b200 import OddSth, _lib
    k = OddSth(h=h).fit(X)
    b = k.X.block
    N = b.n_graphs
    times = []
    with _lib.engine() as eng:
        eng.pack(b.graph_ptr, b.row_ptr, b.col_idx, k.X.ids, None, None)
        for it in range(repeat + 1):
            t0 = time.perf_counter()
            st = eng.odd_features(k.h_, k.X.rank)
            fs = (st.ms_hash, st.ms_columns)
            K, _, _ = eng.gram(N, stats=st, want_diag=False)
            wall = (time.perf_counter() - t0) * 1e3
            if it:
                times.append({"dags+ids": fs[0], "columns": fs[1], "gram": float(sum(st.ms_level_gram)) + st.ms_combine,
                              "d2h": st.ms_d2h, "wall": wall})
    med = {key: float(np.median([t[key] for t in times])) for key in times[0]}
    out = {"workload": name, "h": h, "graphs": N, "vertices": int(b.graph_ptr[-1]), "directed_edges": int(len(b.col_idx)),
           "identities": int(st.n_columns), "bit_planes": int(st.n_levels), "node_slots": int(st.n_entries),
           "hash_retries": int(st.hash_retries), "median_ms": med, "K_checksum": float(np.sum(K)),
           "reference_host": reference_time(X, ref_prefix, h)}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--ref-prefix", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from bench import gen_list
    from odd_cases import mutag
    result = {"card": card(), "runs": []}
    M = mutag()
    G = gen_list(a.n, 40, 0)
    for h in (None, 3):
        result["runs"].append(run("MUTAG", M, h, a.repeat, len(M)))
        result["runs"].append(run("bench.gen_list(%d, 40, 0)" % a.n, G, h, a.repeat, a.ref_prefix))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({"card": result["card"]}))


if __name__ == "__main__":
    main()
