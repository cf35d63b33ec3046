"""WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance and over OddSth, n_iter = 5, on the tools/bench_nspd.py
workload (bench.gen_list(n, 40, 0) with edge label (l_u + l_v) % 3), and the real reference (oracle/_ref) on the host.

    python tools/bench_wl_bases.py [--n 2000] [--repeat 3] [--ref-prefix 40] [--out result.json]

`wall` is the host time of fit_transform (K delivered to the host), median of `repeat` runs after one warm-up run;
`numbering` is the share of it spent numbering the WL classes on the host the reference's way
(wl_reference_dictionaries).  The reference is timed on the first `ref-prefix` graphs and extrapolated linearly in the
number of graphs (a lower bound: its per-level Grams grow faster)."""
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

BASES = {"NSPD": ("NeighborhoodSubgraphPairwiseDistance", {}), "ODD": ("OddSth", {})}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def workload(n):
    from bench import gen_list
    return [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in gen_list(n, 40, 0)]


def reference_time(name, X, prefix):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.isdir(os.path.join(ref, "grakel")):
        return None
    sys.path.insert(0, ref)
    import grakel.kernels as gk
    prefix = min(prefix, len(X))
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gk.WeisfeilerLehman(n_iter=5, base_graph_kernel=getattr(gk, BASES[name][0])).fit_transform(X[:prefix])
    dt = time.perf_counter() - t0
    return {"graphs": prefix, "seconds": dt, "extrapolated_s_linear_in_graphs": dt * len(X) / prefix}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--ref-prefix", type=int, default=40)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import grakel_b200
    X = workload(a.n)
    res = {"card": card(), "graphs": a.n, "n_iter": 5}
    for name, (cls, params) in BASES.items():
        base = getattr(grakel_b200, cls)
        walls, numbering = [], []
        for i in range(a.repeat + 1):
            k = grakel_b200.WeisfeilerLehman(n_iter=5, base_graph_kernel=(base, dict(params)))
            t0 = time.perf_counter()
            k.fit_transform(X)
            if i:
                walls.append((time.perf_counter() - t0) * 1e3)
                numbering.append(k.ms_host_numbering_)
        res[name] = {"wall_ms": float(np.median(walls)), "numbering_ms": float(np.median(numbering)),
                     "numbering_share": float(np.median(numbering) / np.median(walls)),
                     "reference": reference_time(name, X, a.ref_prefix)}
        print(name, json.dumps(res[name]), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
