"""Build tests/golden/wl_sm.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_wl_sm.py
For every case of tests/wl_sm_cases.py and each of its n_iter values, WeisfeilerLehman over SubgraphMatching: K of
fit_transform with diagonal(), of a transform after fit_transform and after fit (the transformed graphs carry labels
the fitted ones do not) with diagonal(), normalize off and on.  Every error case keeps the exception's type and
message."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import wl_sm_cases as cases  # noqa: E402
from grakel import Graph  # noqa: E402
from grakel.kernels import SubgraphMatching, WeisfeilerLehman  # noqa: E402


def record(out, key, fn):
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            val = fn()
        if isinstance(val, tuple):
            out[key + "_x"], out[key + "_y"] = (np.asarray(v, dtype=np.float64) for v in val)
        else:
            out[key] = np.asarray(val, dtype=np.float64)
    except Exception as e:  # noqa: BLE001
        out[key + "_error"] = np.array([type(e).__name__, str(e)])


def main():
    out = {}
    for name, (X, Y, params, n_iters) in cases.cases().items():
        if name in cases.GRAPH_OBJECT_CASES:
            X, Y = [Graph(*x) for x in X], [Graph(*y) for y in Y]
        for n_iter in n_iters:
            def wl(normalize):
                return WeisfeilerLehman(n_iter=n_iter, normalize=normalize,
                                        base_graph_kernel=(SubgraphMatching, dict(params)))
            for norm in (False, True):
                tag = "%s_%d%s" % (name, n_iter, "_norm" if norm else "")
                k = wl(norm)
                record(out, tag + "_fit_transform", lambda: k.fit_transform(X))
                record(out, tag + "_ft_diag", lambda: k.diagonal())
                record(out, tag + "_ft_transform", lambda: k.transform(Y))
                k = wl(norm)
                record(out, tag + "_fit_transform_y", lambda: k.fit(X).transform(Y))
                record(out, tag + "_fit_diag", lambda: k.diagonal())
            print(name, n_iter, "done", flush=True)
    for name, (X, params) in cases.error_cases().items():
        record(out, "err_" + name, lambda: WeisfeilerLehman(
            n_iter=2, base_graph_kernel=(SubgraphMatching, dict(params))).fit_transform(X))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "wl_sm.npz"), **out)


if __name__ == "__main__":
    main()
