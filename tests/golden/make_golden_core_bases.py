"""Build tests/golden/core_bases.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_core_bases.py
For every base of tests/core_bases_cases.py, CoreFramework's K of fit_transform and of fit + transform (the new graphs
carry labels the fitted ones do not, and reach a higher maximum core), normalize off and on, the transform after a
fit_transform as well as after a fit, diagonal() after each (a tuple is stored as key_0, key_1), a set with a graph that
is one isolated vertex (fit_transform, and fit then transform), and a fit set without edge labels.  NeighborhoodHash
also runs with one RandomState shared by the levels and with numpy's global stream (seeded before every case).  A
case whose reference call raises stores the exception's type and message instead."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import core_bases_cases as cases  # noqa: E402
from grakel.kernels import (CoreFramework, NeighborhoodHash, OddSth, SubgraphMatching,  # noqa: E402
                            WeisfeilerLehmanOptimalAssignment)

KINDS = {"NH": NeighborhoodHash, "ODD": OddSth, "WLOA": WeisfeilerLehmanOptimalAssignment, "SM": SubgraphMatching}


def record(out, key, fn):
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            res = fn()
        if isinstance(res, tuple):
            for i, r in enumerate(res):
                out[key + "_%d" % i] = np.asarray(r, dtype=np.float64)
        else:
            out[key] = np.asarray(res, dtype=np.float64)
    except Exception as e:  # noqa: BLE001
        out[key + "_error"] = np.array([type(e).__name__, str(e)])


def main():
    X, Y, Z, U = cases.fit_set(), cases.transform_set(), cases.isolated_set(), cases.unlabelled_edges_set()
    out = {}
    for name in cases.BASES:
        def core(normalize):
            np.random.seed(cases.GLOBAL_SEED)
            kind, params = cases.params_of(name)
            return CoreFramework(normalize=normalize, base_graph_kernel=(KINDS[kind], params))
        for norm in (False, True):
            tag = name + ("_norm" if norm else "")

            for key, data in (("_fit_transform", X), ("_isolated", Z)):
                k = core(norm)
                record(out, tag + key, lambda: k.fit_transform(data))
                record(out, tag + key + "_diag", k.diagonal)

            k = core(norm)
            record(out, tag + "_ft_transform", lambda: (k.fit_transform(X), k.transform(Y))[1])
            record(out, tag + "_ft_transform_diag", k.diagonal)

            k = core(norm)
            record(out, tag + "_fit_transform_y", lambda: k.fit(X).transform(Y))
            record(out, tag + "_fit_transform_y_diag", k.diagonal)

            k = core(norm)
            record(out, tag + "_isolated_fit", lambda: k.fit(Z).transform(X))
            k = core(norm)
            record(out, tag + "_unlabelled_edges_fit", lambda: k.fit(U).transform(Y))
        print(name, sorted(k for k in out if k.startswith(name)), flush=True)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "core_bases.npz"), **out)


if __name__ == "__main__":
    main()
