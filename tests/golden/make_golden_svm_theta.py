"""Build tests/golden/svm_theta.npz from the real reference (oracle/_ref, installed by oracle/build_ref.sh).

Run from the repository root:  python tests/golden/make_golden_svm_theta.py
Every case of tests/svmt_cases.py stores its inputs, the reference's K of fit_transform and transform with normalize
off and on, and per fitted and transformed graph what the reference's own run produced: the smallest eigenvalue m its
`eigvalsh` returned, the alphas its `_calculate_svm_theta_` returned, the n_iter_ of its OneClassSVM fit, the samples
per subset size its `distribute_samples` returned, the index arrays `choice` drew (from a recording RandomState), phi,
and the MT19937 state after the fit and after the transform.  The error cases store the exception the reference
raises."""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import svmt_cases  # noqa: E402


class Recording(np.random.RandomState):
    """A RandomState that keeps every index array `choice` returns."""

    def __init__(self, seed):
        super().__init__(seed)
        self.drawn = []

    def choice(self, *args, **kwargs):
        out = super().choice(*args, **kwargs)
        self.drawn.append(np.asarray(out))
        return out


def _pack_graphs(out, key, G):
    out[key + "_sizes"] = np.array([A.shape[0] for A in G], dtype=np.int64)
    out[key + "_adj"] = np.concatenate([np.asarray(A, dtype=np.float64).ravel() for A in G])


def _per_graph(out, key, rec, lo, L, phis, drawn):
    out[key + "_m"] = np.array(rec["m"])
    out[key + "_alpha"] = np.concatenate(rec["alpha"])
    out[key + "_iters"] = np.array(rec["iters"], dtype=np.int64)
    sched = np.zeros((len(rec["sched"]), L), dtype=np.int64)
    for g, d in enumerate(rec["sched"]):
        for level, v in d.items():
            sched[g, level - lo] = v
    out[key + "_sched"] = sched
    out[key + "_phi"] = np.array([p[:, 0] for p in phis])
    out[key + "_drawn"] = (np.concatenate(drawn) if drawn else np.zeros(0)).astype(np.uint8)
    out[key + "_drawn_len"] = np.array([len(d) for d in drawn], dtype=np.int64)


def _state(out, key, rs):
    _, mt_key, pos, _, _ = rs.get_state()
    out[key + "_key"] = np.asarray(mt_key, dtype=np.uint32)
    out[key + "_pos"] = np.array(pos, dtype=np.int64)


def main():
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))
    from grakel import GraphKernel
    from grakel.datasets.testing import generate_dataset
    from grakel.graph import Graph
    from grakel.kernels import SvmTheta as Ref
    from grakel.kernels import svm_theta as ref_module
    from nspd_cases import mutag as mutag_sets

    # what the reference computes per graph, taken from its own calls
    rec = {"m": [], "alpha": [], "iters": [], "sched": []}

    def eigvalsh(*a, **k):
        w = ref_eigvalsh(*a, **k)
        rec["m"].append(float(w[0]))
        return w

    def calculate(A):
        alphas = ref_calculate(A)
        rec["alpha"].append(np.array(alphas))
        return alphas

    def distribute(*a):
        d = ref_distribute(*a)
        rec["sched"].append(dict(d))
        return d

    class OneClass(ref_module.OneClassSVM):
        def fit(self, *a, **k):
            out = super().fit(*a, **k)
            rec["iters"].append(int(np.asarray(self.n_iter_).reshape(-1)[0]))
            return out

    ref_eigvalsh, ref_calculate, ref_distribute = (ref_module.eigvalsh, ref_module._calculate_svm_theta_,
                                                   ref_module.distribute_samples)
    ref_module.eigvalsh, ref_module._calculate_svm_theta_ = eigvalsh, calculate
    ref_module.distribute_samples, ref_module.OneClassSVM = distribute, OneClass

    class Rec(Ref):
        def parse_input(self, X):
            for v in rec.values():
                v.clear()
            phis = super().parse_input(X)
            self.parsed_.append((phis, {q: list(v) for q, v in rec.items()}))
            return phis

    wrap = lambda G: [[A] for A in G]
    mutag = [Graph(e, {}, {}, "adjacency").get_adjacency_matrix().astype(float) for e, _, _ in mutag_sets()]
    out = {}
    all_cases = svmt_cases.cases(generate_dataset, mutag)
    by_name = {c[0]: c for c in all_cases}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for name, X, Y, params in all_cases:
            _pack_graphs(out, name + "/x", X)
            _pack_graphs(out, name + "/y", Y)
            for norm in (False, True):
                p = dict(params)
                rs = Recording(p.pop("random_state"))
                k = Rec(normalize=norm, random_state=rs, **p)
                k.parsed_ = []
                out[f"{name}/fit/{int(norm)}"] = k.fit_transform(wrap(X))
                n_fit_draws = len(rs.drawn)
                if not norm:
                    _state(out, name + "/state_fit", rs)
                out[f"{name}/transform/{int(norm)}"] = k.transform(wrap(Y))
                if not norm:
                    _state(out, name + "/state_transform", rs)
                    lo, hi = k.subsets_size_range
                    for key, (phis, r), drawn in (("xg", k.parsed_[0], rs.drawn[:n_fit_draws]),
                                                  ("yg", k.parsed_[1], rs.drawn[n_fit_draws:])):
                        _per_graph(out, name + "/" + key, r, lo, hi - lo + 1, phis, drawn)
        # a second fit continues the random stream
        name, base, params = svmt_cases.SECOND_FIT
        X, Y = by_name[base][1], by_name[base][2]
        k = Ref(**params)
        k.fit(wrap(X))
        out[name + "/fit/0"] = k.fit_transform(wrap(X))
        out[name + "/transform/0"] = k.transform(wrap(Y))
        # GraphKernel forwards random_state
        for name, base, params in (svmt_cases.GRAPH_KERNEL, svmt_cases.GRAPH_KERNEL_DICT):
            X, Y = by_name[base][1], by_name[base][2]
            gk = GraphKernel(**params)
            out[name + "/fit/0"] = gk.fit_transform(wrap(X))
            out[name + "/transform/0"] = gk.transform(wrap(Y))
        # a user metric goes through the pairwise driver
        name, base, params = svmt_cases.CUSTOM_METRIC
        X, Y = by_name[base][1], by_name[base][2]
        for norm in (False, True):
            k = Ref(normalize=norm, **params)
            out[f"{name}/fit/{int(norm)}"] = k.fit_transform(wrap(X))
            out[f"{name}/transform/{int(norm)}"] = k.transform(wrap(Y))
        # ZeroDivisionError after the draws of the graphs before the small one
        name, X, params = svmt_cases.ZERO_DIVISION
        rs = np.random.RandomState(params["random_state"])
        try:
            Ref(random_state=rs).fit(wrap(X))
        except ZeroDivisionError:
            _state(out, name + "/state", rs)
        else:
            raise AssertionError("the reference did not raise ZeroDivisionError")
        for name, params in svmt_cases.ERROR_CASES:
            try:
                Ref(**params).fit([[np.ones((3, 3))]])
                out["error/" + name] = np.array("none")
            except Exception as e:  # noqa: BLE001 - the type is the golden
                out["error/" + name] = np.array(type(e).__name__)
    np.savez_compressed(svmt_cases.GOLDEN, **out)
    print("wrote", svmt_cases.GOLDEN, len(out), "arrays")


if __name__ == "__main__":
    main()
