"""Build tests/golden/graphlet_sampling.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_graphlet_sampling.py
Every case of tests/gs_cases.py stores its graphs, the reference's K of fit_transform and transform with normalize off
and on, its diagonal() after the transform, the MT19937 state after the fit and after the transform, and the index
arrays `choice` drew (from a recording RandomState).  The error cases store the exception the reference raises."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
import gs_cases  # noqa: E402
from grakel import Graph  # noqa: E402
from grakel.kernels import GraphletSampling  # noqa: E402


class Recording(np.random.RandomState):
    """A RandomState that keeps every index array `choice` returns."""

    def __init__(self, seed):
        super().__init__(seed)
        self.drawn = []

    def choice(self, *args, **kwargs):
        out = super().choice(*args, **kwargs)
        self.drawn.append(np.asarray(out))
        return out


def _pack(out, key, G):
    out[key + "_sizes"] = np.array([A.shape[0] for A in G], dtype=np.int64)
    out[key + "_adj"] = np.concatenate([A.ravel() for A in G]) if G else np.zeros(0)


def main():
    out = {}
    for name, gname, k, sampling, form, seed in gs_cases.CASES:
        X, Y = gs_cases.graphs(gname, seed)
        _pack(out, name + "_X", X)
        _pack(out, name + "_Y", Y)
        Xi = [gs_cases.element(A, form, Graph) for A in X]
        Yi = [gs_cases.element(A, form, Graph) for A in Y]
        for norm in (False, True):
            rs = Recording(seed)
            gk = GraphletSampling(k=k, sampling=dict(sampling), random_state=rs, normalize=norm)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                Kf = gk.fit_transform(Xi)
                st_fit = rs.get_state()
                n_fit_draws = len(rs.drawn)
                Kt = gk.transform(Yi)
                xd, yd = gk.diagonal()
            st = rs.get_state()
            tag = "%s_n%d" % (name, norm)
            out[tag + "_Kf"] = Kf
            out[tag + "_Kt"] = Kt
            out[tag + "_xdiag"] = np.asarray(xd, dtype=np.float64)
            out[tag + "_ydiag"] = np.asarray(yd, dtype=np.float64)
            out[tag + "_mt_fit"] = np.array(st_fit[1], dtype=np.uint32)
            out[tag + "_pos_fit"] = np.array(st_fit[2])
            out[tag + "_mt"] = np.array(st[1], dtype=np.uint32)
            out[tag + "_pos"] = np.array(st[2])
            if not norm:
                d = rs.drawn
                out[name + "_drawn_sizes"] = np.array([len(a) for a in d], dtype=np.int64)
                out[name + "_drawn"] = np.concatenate(d).astype(np.int64) if d else np.zeros(0, dtype=np.int64)
                out[name + "_n_fit_draws"] = np.array(n_fit_draws)
        print(name, Kf.shape, Kt.shape)
    X, _ = gs_cases.graphs("small", 1)
    for name, params in gs_cases.ERROR_CASES:
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                GraphletSampling(**params).fit([[A] for A in X])
            raise AssertionError(name + " did not raise")
        except Exception as e:  # noqa: BLE001
            out["err_" + name] = np.array([type(e).__name__, str(e)])
            print(name, type(e).__name__, e)
    np.savez_compressed(gs_cases.GOLDEN, **out)


if __name__ == "__main__":
    main()
