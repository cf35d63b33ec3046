"""A/B measurement of the Gram GEMM's head panel type: u8 (u8 x u8 -> s32 wgmma, the default) against bf16
(GRAKEL_B200_U8=0), in one process on one GPU.

  python tools/bench_u8_gram.py [--rounds R] [--steps K] [--out FILE]

Prints (and writes to FILE as JSON, if given):
  gpu          card name, power limit and maximum SM clock (nvidia-smi), read in this run
  config2      BASELINE config 2 (10 000 graphs, h = 5, one gk_wl_gram pass per step, fp32 K on the device): the two
               modes alternate round by round, a separate handle each; ms per pass and the stage split per round
  dense        the dense-mode rate: every shared column in the panel (GK_DENSE_ALL), N (N + 1) D_c / GEMM time, in
               T(FL)OP/s, beside the data-sheet dense figures (989 bf16, 1 979 int8 -- for a 700 W card)
  sweep        ms per pass at a forced head/tail threshold (GRAKEL_B200_FORCE_T = 8 ... 256) in both modes, and the
               threshold the cost model chose by itself
  config3/wloa ShortestPath (config 3) and WL-OA on the graphs of config 2, both modes
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (workload generators only; bench.main is not run)

DATASHEET = {"bf16": 989.0, "u8": 1979.0}
MODES = (("bf16", "0"), ("u8", "1"))


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return dict(zip(q.split(","), [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]))
    except Exception as e:  # pragma: no cover
        return {"error": repr(e)}


def set_mode(flag):
    os.environ["GRAKEL_B200_U8"] = flag


def timed(eng, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    stages = []
    eng.event_record(0)
    for _ in range(steps):
        st = fn()
        stages.append((st.ms_features, st.ms_panel, st.ms_gemm, st.ms_tail))
    eng.event_record(1)
    eng.sync()
    s = np.mean(np.asarray(stages), axis=0)
    return eng.event_elapsed(0, 1) / steps, {"features": s[0], "columns+panel": s[1], "gram_gemm": s[2], "tail": s[3]}, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out")
    args = ap.parse_args()
    from grakel_b200 import _lib
    res = {"gpu": gpu_info()}
    print(json.dumps(res["gpu"]), flush=True)

    gp, rp, ci, lab = bench.pack_workload(bench.N_GRAPHS)
    n = len(gp) - 1
    H = bench.H
    engs = {}
    for name, flag in MODES:
        set_mode(flag)
        e = _lib.Engine(0)
        e.pack(gp, rp, ci, lab)
        engs[name] = e

    def c2(e):
        return lambda: e.wl_gram(H, out=False, dtype=np.float32)[2]

    # ---- config 2, alternating modes
    rows = {name: [] for name, _ in MODES}
    for r in range(args.rounds):
        for name, flag in MODES:
            set_mode(flag)
            ms, stages, st = timed(engs[name], c2(engs[name]), args.steps, 200 if r == 0 else 20)
            rows[name].append({"ms_per_pass": ms, "stages_ms": stages, "T": int(st.threshold),
                               "head_columns": int(st.n_dense_columns), "gemm_elem_bytes": int(st.gemm_elem_bytes),
                               "gemm_launches": int(st.gemm_launches)})
            print("config2 %-4s round %d: %.4f ms/pass  %s  T %d Dc %d elem %d" % (
                name, r, ms, {k: round(v, 4) for k, v in stages.items()}, st.threshold, st.n_dense_columns,
                st.gemm_elem_bytes), flush=True)
    res["config2"] = {name: {"rounds": rows[name], "median_ms": float(np.median([x["ms_per_pass"] for x in rows[name]])),
                             "min_ms": float(np.min([x["ms_per_pass"] for x in rows[name]])),
                             "max_ms": float(np.max([x["ms_per_pass"] for x in rows[name]])),
                             "median_gemm_ms": float(np.median([x["stages_ms"]["gram_gemm"] for x in rows[name]]))}
                      for name, _ in MODES}

    # ---- dense-mode rate (every shared column dense)
    res["dense"] = {}
    for name, flag in MODES:
        set_mode(flag)
        e = engs[name]
        ms, stages, st = timed(e, lambda: e.wl_gram(H, out=False, dtype=np.float32, dense_all=True)[2], 20, 5)
        gemm = []
        for _ in range(20):
            gemm.append(e.wl_gram(H, out=False, dtype=np.float32, dense_all=True)[2].ms_gemm)
        g = float(np.median(gemm))
        dc = int(st.n_dense_columns)
        rate = float(n) * (n + 1) * dc / (g * 1e-3) / 1e12
        res["dense"][name] = {"head_columns": dc, "gemm_ms": g, "rate_T": rate, "datasheet_T": DATASHEET[name],
                              "gemm_elem_bytes": int(st.gemm_elem_bytes)}
        print("dense %-4s: Dc %d gemm %.4f ms -> %.1f T(FL)OP/s (data sheet %.0f)" % (name, dc, g, rate, DATASHEET[name]),
              flush=True)
    res["dense"]["u8_over_bf16"] = res["dense"]["u8"]["rate_T"] / res["dense"]["bf16"]["rate_T"]
    print("dense u8 / bf16 rate: %.3f" % res["dense"]["u8_over_bf16"], flush=True)

    # ---- forced-threshold sweep
    res["sweep"] = {}
    for name, flag in MODES:
        set_mode(flag)
        e = engs[name]
        sw = {}
        for T in (8, 16, 32, 64, 128, 256):
            os.environ["GRAKEL_B200_FORCE_T"] = str(T)
            ms, stages, st = timed(e, c2(e), 20, 5)
            sw[T] = {"ms_per_pass": ms, "stages_ms": stages, "head_columns": int(st.n_dense_columns)}
            print("sweep %-4s T %4d: %.4f ms/pass gemm %.4f tail %.4f Dc %d" % (
                name, T, ms, stages["gram_gemm"], stages["tail"], st.n_dense_columns), flush=True)
        del os.environ["GRAKEL_B200_FORCE_T"]
        ms, stages, st = timed(e, c2(e), 20, 5)
        sw["model"] = {"T": int(st.threshold), "ms_per_pass": ms}
        print("sweep %-4s cost model: T %d %.4f ms/pass" % (name, st.threshold, ms), flush=True)
        res["sweep"][name] = sw
    for e in engs.values():
        e.close()

    # ---- config 3 and WL-OA
    from grakel_b200.packing import label_ids, pack
    X = bench.gen_list(5000, 60, 0, as_adj=True)
    b3 = pack(X, "sp", want_weights=True)
    ids3, _ = label_ids(b3.labels, None, sort_new=False)
    del X
    X2 = bench.gen_list(n)
    bo = pack(X2, "wloa", len_ok=lambda k: k >= 2)
    idso, _ = label_ids(bo.labels, None, sort_new=True)
    del X2
    res["config3"], res["wloa"] = {}, {}
    for r in range(3):
        for name, flag in MODES:
            set_mode(flag)
            e = _lib.Engine(0)
            e.pack(b3.graph_ptr, b3.row_ptr, b3.col_idx, ids3, b3.weights)

            def s3():
                st = e.sp_features(with_labels=True)
                e.gram(b3.n_graphs, out=False, dtype=np.float32, stats=st, want_diag=False)
                return st
            ms, stages, st = timed(e, s3, 10, 3)
            res["config3"].setdefault(name, []).append({"ms_per_step": ms, "stages_ms": stages,
                                                        "gemm_elem_bytes": int(st.gemm_elem_bytes)})
            print("config3 %-4s: %.4f ms/step %s elem %d" % (name, ms, {k: round(v, 4) for k, v in stages.items()},
                                                             st.gemm_elem_bytes), flush=True)
            e.pack(bo.graph_ptr, bo.row_ptr, bo.col_idx, idso)

            def so():
                st = e.wl_oa_features(H)
                e.gram(bo.n_graphs, out=False, dtype=np.float32, stats=st, want_diag=False)
                return st
            ms, stages, st = timed(e, so, 10, 3)
            res["wloa"].setdefault(name, []).append({"ms_per_step": ms, "stages_ms": stages,
                                                     "gemm_elem_bytes": int(st.gemm_elem_bytes)})
            print("wloa    %-4s: %.4f ms/step %s elem %d" % (name, ms, {k: round(v, 4) for k, v in stages.items()},
                                                             st.gemm_elem_bytes), flush=True)
            e.close()
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1, default=float)
    print(json.dumps({"config2_median_ms": {k: res["config2"][k]["median_ms"] for k, _ in MODES},
                      "config2_median_gemm_ms": {k: res["config2"][k]["median_gemm_ms"] for k, _ in MODES},
                      "dense_u8_over_bf16": res["dense"]["u8_over_bf16"], "gpu": res["gpu"]}))


if __name__ == "__main__":
    main()
