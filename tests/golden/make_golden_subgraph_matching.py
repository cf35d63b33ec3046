"""Build tests/golden/subgraph_matching.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_subgraph_matching.py
Every case (tests/sm_cases.py) stores the reference's K of fit_transform and transform, with normalize off and on,
and every error case the name of the exception the reference raises."""
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from sm_cases import GRAPH_OBJECT_CASES, cases, error_cases  # noqa: E402


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel import Graph
    from grakel.kernels import SubgraphMatching as Ref
    out, meta = {}, []
    for name, X, Y, params in cases():
        if name in GRAPH_OBJECT_CASES:
            X = [Graph(*x) for x in X]
            Y = None if Y is None else [Graph(*y) for y in Y]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for norm in (False, True):
                k = Ref(normalize=norm, **params)
                out[f"{name}/fit/{int(norm)}"] = k.fit_transform(X)
                if Y is not None:
                    out[f"{name}/transform/{int(norm)}"] = k.transform(Y)
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
    out["__cases__"] = np.array(json.dumps(meta))
    out["__errors__"] = np.array(json.dumps(errors))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "subgraph_matching.npz"), **out)


if __name__ == "__main__":
    main()
