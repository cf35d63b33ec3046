"""Build tests/golden/hc_bases.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_hc_bases.py
For every case of tests/hc_bases_cases.py and each of its n_iter values, HadamardCode over SubgraphMatching,
PyramidMatch or NeighborhoodSubgraphPairwiseDistance: K of fit_transform with diagonal(), and for every transform set
K of a transform after fit_transform and after fit with diagonal(), normalize off and on.  Every error case keeps the
exception's type and message."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import hc_bases_cases as cases  # noqa: E402
from grakel import Graph  # noqa: E402
from grakel.kernels import (HadamardCode, NeighborhoodSubgraphPairwiseDistance, PyramidMatch,  # noqa: E402
                            SubgraphMatching)

BASES = {"SM": SubgraphMatching, "PM": PyramidMatch, "NSPD": NeighborhoodSubgraphPairwiseDistance}


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
    for name, (base, X, Ys, params, n_iters) in cases.cases().items():
        if name in cases.GRAPH_OBJECT_CASES:
            X, Ys = [Graph(*x) for x in X], {t: [Graph(*y) for y in Y] for t, Y in Ys.items()}
        for n_iter in n_iters:
            def hc(normalize):
                return HadamardCode(n_iter=n_iter, normalize=normalize, base_graph_kernel=(BASES[base], dict(params)))
            for norm in (False, True):
                tag = "%s_%d%s" % (name, n_iter, "_norm" if norm else "")
                k = hc(norm)
                record(out, tag + "_fit_transform", lambda: k.fit_transform(X))
                record(out, tag + "_ft_diag", lambda: k.diagonal())
                for t, Y in sorted(Ys.items()):
                    k = hc(norm)
                    record(out, "%s_%s_ft_transform" % (tag, t), lambda: (k.fit_transform(X), k.transform(Y))[1])
                    k = hc(norm)
                    record(out, "%s_%s_fit_transform_y" % (tag, t), lambda: k.fit(X).transform(Y))
                    record(out, "%s_%s_fit_diag" % (tag, t), lambda: k.diagonal())
            print(name, n_iter, "done", flush=True)
    for name, (base, X, params) in cases.error_cases().items():
        record(out, "err_" + name, lambda: HadamardCode(
            n_iter=2, base_graph_kernel=(BASES[base], dict(params))).fit_transform(X))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "hc_bases.npz"), **out)


if __name__ == "__main__":
    main()
