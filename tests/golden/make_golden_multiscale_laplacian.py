"""Build tests/golden/multiscale_laplacian.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_multiscale_laplacian.py
Every case (tests/ml_cases.py) stores its input graphs, the reference's K of fit_transform and transform with
normalize off and on, the (graph, vertex) samples of every level, the raw (v, w) of every eig call of the fit and its
eigenvalues' distance to the truncation boundary; the error cases store the name of the exception."""
import json
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from ml_cases import ERROR_CASES, generated_cases  # noqa: E402



class RecordingState(np.random.RandomState):
    def __init__(self, seed):
        super().__init__(seed)
        self.lists = []

    def shuffle(self, x):
        super().shuffle(x)
        self.lists.append(list(x))


def boundary_gap(v, P):
    """Smallest relative distance of the sorted eigenvalues to the cut: lambda_P vs lambda_P+1, and any to 1e-6."""
    s = np.sort(np.real(v))[::-1]
    scale = max(abs(s[0]), 1e-300)
    g = np.min(np.abs(s - 1e-6)) / scale
    if len(s) > P:
        g = min(g, abs(s[P - 1] - s[P]) / scale)
    return g


def pack(prefix, els, out):
    out[prefix + "_n"] = np.array([A.shape[0] for A, _ in els], dtype=np.int64)
    out[prefix + "_A"] = np.concatenate([A.ravel() for A, _ in els])
    out[prefix + "_phi"] = np.concatenate([np.asarray(p).reshape(A.shape[0], -1) for A, p in els])


def as_input(els):
    return [[A, {i: list(p[i]) for i in range(A.shape[0])}] for A, p in els]


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    import grakel.kernels.multiscale_laplacian as mlmod
    from grakel import GraphKernel
    from grakel.datasets.testing import generate_dataset
    Ref = mlmod.MultiscaleLaplacian
    out, meta = {}, {"cases": [], "errors": {}}
    real_eig = mlmod.eig
    for name, X, Y, params in generated_cases(generate_dataset):
        pack(name + "/X", X, out)
        pack(name + "/Y", Y, out)
        seed = params["random_state"]
        calls = []

        def rec_eig(K):
            v, w = real_eig(K)
            calls.append((v, w))
            return v, w
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            mlmod.eig = rec_eig
            for norm in (False, True):
                calls.clear()
                rs = RecordingState(seed)
                k = Ref(normalize=norm, **dict(params, random_state=rs))
                out[name + "/K_fit" + ("_norm" if norm else "")] = k.fit_transform(as_input(X))
                out[name + "/K_tr" + ("_norm" if norm else "")] = k.transform(as_input(Y))
            ns = min(sum(A.shape[0] for A, _ in X), params.get("n_samples", 50))
            P = params.get("P", 10)
            gaps = []
            for l, (v, w) in enumerate(calls):
                out[name + "/eig_v_%d" % l] = v
                out[name + "/eig_w_%d" % l] = w
                out[name + "/samples_%d" % l] = np.array(rs.lists[l][:ns], dtype=np.int64)
                gaps.append(float(boundary_gap(v, P)))
            # a second fit on the same estimator (the normalising one) draws new samples
            out[name + "/K_refit"] = k.fit_transform(as_input(X))
            if name == "reference_tests":
                gk = GraphKernel(kernel="ML", random_state=7)
                out[name + "/K_graphkernel"] = gk.fit_transform(as_input(X))
            mlmod.eig = real_eig
        meta["cases"].append({"name": name, "params": {k: v for k, v in params.items()}, "levels": params.get("L", 3) + 1,
                              "gaps": gaps})
    X0 = generated_cases()[0][1]
    for name, params in ERROR_CASES:
        X = as_input(X0)
        if name == "int_labels":
            X = [[A, {i: 1 for i in range(A.shape[0])}] for A, _ in X0]
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                Ref(**params).fit_transform(X)
            meta["errors"][name] = None
        except Exception as e:  # noqa: BLE001
            meta["errors"][name] = type(e).__name__
    out["meta"] = np.array(json.dumps(meta))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "multiscale_laplacian.npz"), **out)
    print(json.dumps(meta, indent=1))


if __name__ == "__main__":
    main()
