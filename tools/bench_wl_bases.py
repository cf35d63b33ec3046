"""WeisfeilerLehman over NeighborhoodSubgraphPairwiseDistance, OddSth and SubgraphMatching (k = 3 and 5), n_iter = 5,
on the tools/bench_nspd.py workload (bench.gen_list(n, 40, 0) with edge label (l_u + l_v) % 3), and the real reference
(oracle/_ref) on the host.

    python tools/bench_wl_bases.py [--n 2000] [--repeat 3] [--ref-prefix 40] [--bases NSPD,ODD,SM] [--out result.json]

`wall` is the host time of fit_transform (K delivered to the host), median of `repeat` runs after one warm-up run;
`numbering` is the share of it spent numbering the WL classes on the host the reference's way
(wl_reference_dictionaries).  The reference is timed on the first `ref-prefix` graphs and extrapolated linearly in the
number of graphs (a lower bound: its per-level Grams grow faster).  For SubgraphMatching the one-pass route is timed
against the per-level device route (n_iter + 1 SubgraphMatching fit_transforms on the level-labelled graphs, the WL
levels computed on the host as tests/wl_sm_oracle.py does and not timed), the two alternated in the same call;
`--ref-prefix 0` skips the reference."""
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
SM_KS = (3, 5)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True).strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def workload(n):
    from bench import gen_list
    return [[g, L, {(u, v): (L[u] + L[v]) % 3 for (u, v) in g}] for g, L in gen_list(n, 40, 0)]


def reference_time(name, X, prefix, params=None):
    ref = os.path.join(ROOT, "oracle", "_ref")
    if prefix <= 0 or not os.path.isdir(os.path.join(ref, "grakel")):
        return None
    sys.path.insert(0, ref)
    import grakel.kernels as gk
    prefix = min(prefix, len(X))
    base = getattr(gk, BASES[name][0] if name in BASES else "SubgraphMatching")
    t0 = time.perf_counter()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        gk.WeisfeilerLehman(n_iter=5, base_graph_kernel=(base, dict(params or {}))).fit_transform(X[:prefix])
    dt = time.perf_counter() - t0
    return {"graphs": prefix, "seconds": dt, "extrapolated_s_linear_in_graphs": dt * len(X) / prefix}


def sm_times(X, k, repeat):
    """(one-pass ms, per-level device ms): medians of `repeat` alternated runs after one warm-up run of each; the
    two K are checked equal."""
    import grakel_b200
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from wl_sm_oracle import level_elements
    levels = [lx for lx, _ in level_elements(X, None, 5)]
    one, per = [], []
    for i in range(repeat + 1):
        t0 = time.perf_counter()
        K1 = grakel_b200.WeisfeilerLehman(n_iter=5, base_graph_kernel=(grakel_b200.SubgraphMatching, {"k": k})
                                          ).fit_transform(X)
        t1 = time.perf_counter()
        K2 = np.sum([grakel_b200.SubgraphMatching(k=k).fit_transform(lx) for lx in levels], axis=0)
        t2 = time.perf_counter()
        if not np.array_equal(K1, K2):
            raise SystemExit("one-pass and per-level K differ at k = %d" % k)
        if i:
            one.append((t1 - t0) * 1e3)
            per.append((t2 - t1) * 1e3)
    return float(np.median(one)), float(np.median(per))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--ref-prefix", type=int, default=40)
    ap.add_argument("--bases", default="NSPD,ODD,SM")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import grakel_b200
    X = workload(a.n)
    res = {"card": card(), "graphs": a.n, "n_iter": 5}
    bases = a.bases.split(",")
    for k in SM_KS if "SM" in bases else ():
        one, per = sm_times(X, k, a.repeat)
        res["SM_k%d" % k] = {"one_pass_ms": one, "per_level_device_ms": per, "per_level_over_one_pass": per / one,
                             "reference": reference_time("SM", X, a.ref_prefix, {"k": k})}
        print("SM k=%d" % k, json.dumps(res["SM_k%d" % k]), flush=True)
    for name, (cls, params) in BASES.items():
        if name not in bases:
            continue
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
