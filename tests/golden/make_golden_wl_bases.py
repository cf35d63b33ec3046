"""Build tests/golden/wl_bases.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_wl_bases.py
For every base of tests/wl_bases_cases.py (NeighborhoodSubgraphPairwiseDistance at three (r, d), OddSth at h = None
and h = 2) and n_iter 1, 2, 5, WeisfeilerLehman's K of fit_transform and of fit + transform (the transformed graphs
carry labels the fitted ones do not), normalize off and on, the transform after a fit_transform as well as after a
fit.  A case whose reference call raises stores the exception's type and message instead."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import wl_bases_cases as cases  # noqa: E402
from grakel.kernels import NeighborhoodSubgraphPairwiseDistance, OddSth, WeisfeilerLehman  # noqa: E402

KINDS = {"NSPD": NeighborhoodSubgraphPairwiseDistance, "ODD": OddSth}


def record(out, key, fn):
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out[key] = np.asarray(fn(), dtype=np.float64)
    except Exception as e:  # noqa: BLE001
        out[key + "_error"] = np.array([type(e).__name__, str(e)])


def main():
    X, Y = cases.fit_set(), cases.transform_set()
    out = {}
    for name, (kind, params) in cases.BASES.items():
        for n_iter in cases.N_ITERS:
            def wl(normalize):
                return WeisfeilerLehman(n_iter=n_iter, normalize=normalize,
                                        base_graph_kernel=(KINDS[kind], dict(params)))
            key = "%s_%d" % (name, n_iter)
            for norm in (False, True):
                tag = key + ("_norm" if norm else "")
                record(out, tag + "_fit_transform", lambda: wl(norm).fit_transform(X))

                def ft_then_t():
                    k = wl(norm)
                    k.fit_transform(X)
                    return k.transform(Y)
                record(out, tag + "_ft_transform", ft_then_t)

                def fit_then_t():
                    k = wl(norm)
                    k.fit(X)
                    return k.transform(Y)
                record(out, tag + "_fit_transform_y", fit_then_t)
            print(key, "done", flush=True)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "wl_bases.npz"), **out)


if __name__ == "__main__":
    main()
