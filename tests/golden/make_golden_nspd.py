"""Build tests/golden/nspd.npz from the real reference (oracle/_ref, installed by __graft_entry__.build()).

Run from the repository root with PYTHONHASHSEED=0:  PYTHONHASHSEED=0 python tests/golden/make_golden_nspd.py
Every case (tests/nspd_cases.py) stores the reference's K of fit_transform and transform, with normalize off and on,
and H[rho, v] of every fitted vertex ([r + 1, vertices] u32, graph after graph), recorded from the reference's own
_hash_neighborhoods."""
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from nspd_cases import GRAPH_OBJECT_CASES, cases  # noqa: E402


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel import Graph
    from grakel.kernels import NeighborhoodSubgraphPairwiseDistance as Ref
    recorded = []
    hash_nb = Ref._hash_neighborhoods

    def record(self, vertices, *args):
        H = hash_nb(self, vertices, *args)
        recorded.append(np.array([[H[rho, v] for v in range(len(vertices))] for rho in range(self.r + 1)],
                                 dtype=np.uint32).reshape(self.r + 1, len(vertices)))
        return H

    Ref._hash_neighborhoods = record
    out = {}
    meta = []
    for name, X, Y, params in cases():
        if name in GRAPH_OBJECT_CASES:
            X = [Graph(*x) for x in X]
            Y = None if Y is None else [Graph(*y) for y in Y]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            for norm in (False, True):
                k = Ref(normalize=norm, **params)
                del recorded[:]
                out[f"{name}/fit/{int(norm)}"] = k.fit_transform(X)
                out[f"{name}/H"] = np.concatenate(recorded, axis=1)
                if Y is not None:
                    out[f"{name}/transform/{int(norm)}"] = k.transform(Y)
        meta.append(name)
    out["__cases__"] = np.array(json.dumps(meta))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "nspd.npz"), **out)


if __name__ == "__main__":
    main()
