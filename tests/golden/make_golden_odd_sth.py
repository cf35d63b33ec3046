"""Build tests/golden/odd_sth.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_odd_sth.py
Every case (tests/odd_cases.py) stores the reference's K of fit_transform and transform, with normalize off and on
(off only for RAW_ONLY_CASES),
the digests of the fitted feature keys (except for KEYLESS_CASES) (identity strings, odd_cases.key_hash) with their C, and every error case the name of the exception the reference
raises."""
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from odd_cases import GRAPH_OBJECT_CASES, KEYLESS_CASES, RAW_ONLY_CASES, cases, error_cases, key_hash  # noqa: E402


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel import Graph
    from grakel.kernels import OddSth as Ref
    out, meta = {}, []
    for name, X, Y, params in cases():
        if name in GRAPH_OBJECT_CASES:
            X = [Graph(x[0], x[1], {}, "dictionary") for x in X]
            Y = None if Y is None else [Graph(y[0], y[1], {}, "dictionary") for y in Y]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for norm in (False,) if name in RAW_ONLY_CASES else (False, True):
                k = Ref(normalize=norm, **params)
                out[f"{name}/fit/{int(norm)}"] = k.fit_transform(X)
                if not norm and name not in KEYLESS_CASES:
                    D = k.X[0]
                    keys = [D[i][2] for i in range(len(D))]
                    out[f"{name}/keys"] = np.array([key_hash(s) for s in keys], dtype=np.uint64)
                    out[f"{name}/C"] = np.array([D[i][0] for i in range(len(D))], dtype=np.int64)
                if Y is not None:
                    out[f"{name}/transform/{int(norm)}"] = k.transform(Y)
                    xd, yd = k.diagonal()
                    out[f"{name}/xdiag/{int(norm)}"] = np.asarray(xd)
                    out[f"{name}/ydiag/{int(norm)}"] = np.asarray(yd)
        meta.append(name)
        print(name, flush=True)
    errors = {}
    for name, X, params in error_cases():
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                Ref(**params).fit_transform(X)
            errors[name] = None
        except Exception as e:  # noqa: BLE001 -- the type is what the golden keeps
            errors[name] = type(e).__name__
    X = next(c[1] for c in cases() if c[0] == "random")
    for name, fn in (("transform_none", lambda: Ref().fit(X).transform(None)),
                     ("fit_then_normalized_transform", lambda: Ref(normalize=True).fit(X).transform(X[:2]))):
        try:
            fn()
            errors[name] = None
        except Exception as e:  # noqa: BLE001
            errors[name] = type(e).__name__
    out["__cases__"] = np.array(json.dumps(meta))
    out["__errors__"] = np.array(json.dumps(errors))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "odd_sth.npz"), **out)


if __name__ == "__main__":
    main()
